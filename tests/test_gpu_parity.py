"""GPU parity tests proper: the CUDA path, called through the C ABI, against the CPU oracle on the same seeded
inputs, plus the reference's golden scenes rendered by the CUDA path.

Bars (BASELINE.json north_star): visible-object indices, MV/MVP, batches, packed index lists, draw records,
visibility bits, depth, shadow atlas and hi-Z are integer / bit-pattern artefacts and must be IDENTICAL;
shaded HDR pixels must agree within 1e-4 (absolute below 1.0, relative above — the target is HDR) on the f32
shading result, and the rgba16f store within one f16 ulp of that.
"""
import os

import numpy as np
import pytest

from harness import TOL, compare_frame_state, hdr_close
from rend3_b200 import glam
from rend3_b200.backend import CAMERA_VIEWPORT, CB_BAKE, CB_CULL, load_cuda_backend
from rend3_b200.layouts import OBJECT_DTYPE
from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings, per_camera_header
from rend3_b200.scenes import cloud_camera, cube_field_scene, object_cloud_records
from rend3_b200.world import Camera

from oracle import load_oracle_backend

pytestmark = pytest.mark.gpu


@pytest.fixture()
def cuda():
    """A fresh context per test: contexts carry cross-frame state (previous invocations, culling buffers)."""
    b = load_cuda_backend(0)
    yield b
    b.close()


# ------------------------------------------------------------------ object cull + uniform bake
@pytest.mark.parametrize("n", [1, 31, 2048, 2049, 200_000])
def test_cull_bake_matches_oracle(cuda, n):
    rec = object_cloud_records(n, seed=2 + n)
    cam = cloud_camera()
    header = per_camera_header(cam, CAMERA_VIEWPORT, (1920, 1080), 1, n)
    out = {}
    for name, b in (("cuda", cuda), ("oracle", load_oracle_backend())):
        b.set_objects(rec)
        b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE | CB_CULL)
        out[name] = (b.readback_visible(CAMERA_VIEWPORT).copy(), b.readback_object_matrices(CAMERA_VIEWPORT, 0, n).copy())
    vis_c, mat_c = out["cuda"]
    vis_o, mat_o = out["oracle"]
    assert np.array_equal(vis_c, vis_o)
    assert np.all(np.diff(vis_c.astype(np.int64)) > 0), "visible list must be ascending"
    en = rec["enabled"] != 0
    assert np.array_equal(mat_c.view(np.uint32).reshape(n, 32)[en], mat_o.view(np.uint32).reshape(n, 32)[en]), "MV/MVP not bit-identical"
    if n >= 2048:
        assert 0 < len(vis_c) < n


def test_config2_one_million_objects_cull_only_bit_exact(cuda):
    """BASELINE config 2 as stated: 1 M instanced objects, frustum cull only (no bake, no shade), 1 GPU — the visible-index list must be
    IDENTICAL to the oracle's (uniform_prep.wgsl is not run; batching.rs:144-148 + frustum.rs:148-161 are)."""
    n = 1_000_000
    rec = object_cloud_records(n, seed=2)
    header = per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (1920, 1080), 1, n)
    orc = load_oracle_backend()
    for b in (cuda, orc):
        b.set_objects(rec)
        b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_CULL)
    vc, vo = cuda.readback_visible(CAMERA_VIEWPORT), orc.readback_visible(CAMERA_VIEWPORT)
    assert np.array_equal(vc, vo), "config 2: cull indices differ from the oracle"
    assert 0.2 * n < len(vc) < 0.8 * n and np.all(np.diff(vc.astype(np.int64)) > 0)


def test_config4_ten_million_objects_cull_bake_bit_exact(cuda):
    """BASELINE config 4's per-GPU shard at full size: 10 M object records, cull + bake — the visible list AND every MV / MVP word of every
    enabled slot identical to the oracle (2.56 GB of matrices compared word for word)."""
    n = 10_000_000
    rec = object_cloud_records(n, seed=4)
    header = per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (1920, 1080), 1, n)
    orc = load_oracle_backend()
    import oracle
    oracle.set_threads(os.cpu_count() or 1)
    for b in (cuda, orc):
        b.set_objects(rec)
        b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE | CB_CULL)
    assert np.array_equal(cuda.readback_visible(CAMERA_VIEWPORT), orc.readback_visible(CAMERA_VIEWPORT)), "config 4: visible list differs from the oracle"
    en = rec["enabled"] != 0
    chunk = 1_000_000
    for first in range(0, n, chunk):     # chunked so that the host copies stay small
        a = cuda.readback_object_matrices(CAMERA_VIEWPORT, first, chunk).view(np.uint32).reshape(chunk, 32)
        o = orc.readback_object_matrices(CAMERA_VIEWPORT, first, chunk).view(np.uint32).reshape(chunk, 32)
        e = en[first:first + chunk]
        assert np.array_equal(a[e], o[e]), f"config 4: MV/MVP words differ in slots [{first}, {first + chunk})"


def test_cull_only_and_bake_only_modes(cuda):
    n = 50_000
    rec = object_cloud_records(n, seed=11)
    header = per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (1920, 1080), 1, n)
    orc = load_oracle_backend()
    for b in (cuda, orc):
        b.set_objects(rec)
        b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_CULL)
    assert np.array_equal(cuda.readback_visible(CAMERA_VIEWPORT), orc.readback_visible(CAMERA_VIEWPORT))
    for b in (cuda, orc):
        b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE)
    en = rec["enabled"] != 0
    a = cuda.readback_object_matrices(CAMERA_VIEWPORT, 0, n).view(np.uint32).reshape(n, 32)
    o = orc.readback_object_matrices(CAMERA_VIEWPORT, 0, n).view(np.uint32).reshape(n, 32)
    assert np.array_equal(a[en], o[en])


def test_degenerate_records_match_oracle(cuda):
    """NaN / infinite sphere centres and radii, zero radii, huge transforms, disabled slots: the visible list and the baked matrices of
    the enabled slots stay bit-identical (NaNs included) to the oracle."""
    n = 4096
    rec = object_cloud_records(n, seed=13)
    rng = np.random.default_rng(14)
    pick = rng.permutation(n)
    rec["sphere_center"][pick[:64]] = np.nan
    rec["sphere_radius"][pick[64:128]] = np.nan
    rec["sphere_center"][pick[128:192], 0] = np.inf
    rec["sphere_radius"][pick[192:256]] = np.inf
    rec["sphere_radius"][pick[256:320]] = 0.0
    rec["transform"][pick[320:384]] *= np.float32(1e30)
    rec["transform"][pick[384:448], 5] = np.nan
    rec["enabled"][pick[448:512]] = 0
    header = per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (1920, 1080), 1, n)
    orc = load_oracle_backend()
    for b in (cuda, orc):
        b.set_objects(rec)
        b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE | CB_CULL)
    assert np.array_equal(cuda.readback_visible(CAMERA_VIEWPORT), orc.readback_visible(CAMERA_VIEWPORT))
    en = rec["enabled"] != 0
    a = cuda.readback_object_matrices(CAMERA_VIEWPORT, 0, n).view(np.uint32).reshape(n, 32)
    o = orc.readback_object_matrices(CAMERA_VIEWPORT, 0, n).view(np.uint32).reshape(n, 32)
    # NaN payloads may differ between x86 and the GPU: compare numerically with NaN == NaN
    af, of = a[en].view(np.float32), o[en].view(np.float32)
    assert np.array_equal(np.isnan(af), np.isnan(of)) and np.array_equal(a[en][~np.isnan(af)], o[en][~np.isnan(of)])


def test_live_mask_and_update_objects(cuda):
    """Slots that are live but disabled stay in the visible set (batching.rs:144 iterates enumerated objects),
    and r3_update_objects scatters like ScatterCopy."""
    n = 5000
    rec = object_cloud_records(n, seed=5, extent=100.0, disabled_fraction=0.2)
    header = per_camera_header(cloud_camera(pull_back=30.0), CAMERA_VIEWPORT, (640, 480), 1, n)
    live = (np.arange(n) % 7 != 0).astype(np.uint8)
    key = np.zeros(n, dtype=np.uint64)
    loc = rec["sphere_center"].copy()
    orc = load_oracle_backend()
    slots = np.array([3, 77, 4096, 4999, 10_000], dtype=np.uint32)   # last one is out of range -> dropped
    new = object_cloud_records(len(slots), seed=99, extent=100.0, disabled_fraction=0.0)
    for b in (cuda, orc):
        b.set_objects(rec)
        b.set_object_sort_info(key, live | 2, loc)
        b.update_objects(slots, new)
        b.object_uniform_upload(CAMERA_VIEWPORT, header)
    vc, vo = cuda.readback_visible(CAMERA_VIEWPORT), orc.readback_visible(CAMERA_VIEWPORT)
    assert np.array_equal(vc, vo)
    assert not np.any(vc % 7 == 0)
    mc = cuda.readback_object_matrices(CAMERA_VIEWPORT, 0, n).view(np.uint32).reshape(n, 32)
    mo = orc.readback_object_matrices(CAMERA_VIEWPORT, 0, n).view(np.uint32).reshape(n, 32)
    assert np.array_equal(mc[[3, 77, 4096, 4999]], mo[[3, 77, 4096, 4999]])


def test_gpu_skinning_is_bit_exact(cuda):
    """skinning.wgsl on the GPU against the oracle: the whole mesh buffer (skinned positions + normals written into the
    overridden ranges) must be bit-identical — the positions feed the bit-exact cull and raster stages."""
    import skinning_case

    words, inputs, joints, _ = skinning_case.build(seed=2, vertex_counts=(257, 5000, 1), joints_per_skeleton=(3, 16, 1))
    orc = load_oracle_backend()
    for b in (cuda, orc):
        b.set_mesh_buffer(words)
        b.skin(inputs, joints)
    a, o = cuda.readback_mesh_buffer(len(words)), orc.readback_mesh_buffer(len(words))
    assert np.array_equal(a, o)
    assert not np.array_equal(a, words), "skinning must have written the overridden ranges"


# ------------------------------------------------------------------ whole frames
def test_cube_field_frame_matches_oracle(cuda):
    """C1-shaped scene at reduced size: 2000 cubes, directional light with shadow map, 3 point lights."""
    res = (480, 270)
    ev = cube_field_scene(n_objects=2000, seed=1, resolution=res, n_point_lights=3, shadow_resolution=512, pull_back=12.0, extent=30.0)
    orc = load_oracle_backend()
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0), ambient_color=(0.02, 0.02, 0.02, 1.0))
    for b in (cuda, orc):
        BaseRenderGraph(b).add_to_graph(ev, res, 1, settings)
    compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT, 0], what="cube field")
    st = cuda.forward_stats()
    assert st[0] > 0 and st[1] >= st[2] > 0
    for mip in range(0, 9, 2):
        assert np.array_equal(cuda.readback_hiz(mip).view(np.uint32), orc.readback_hiz(mip).view(np.uint32))


def test_multi_frame_predicted_residual(cuda):
    """Three frames with a 0.5 degree yaw step: predicted pass + hi-Z occlusion + residual pass (base.rs:158-172)."""
    res = (320, 200)
    ev = cube_field_scene(n_objects=1500, seed=3, resolution=res, n_dir_lights=0, pull_back=8.0, extent=20.0, subdivisions=(1, 2))
    orc = load_oracle_backend()
    graphs = {id(b): BaseRenderGraph(b) for b in (cuda, orc)}
    from rend3_b200.world import CameraState, LEFT
    base_view = ev.camera.view.copy()
    for frame in range(3):
        view = glam.mul(glam.from_rotation_y(np.float32(np.radians(0.5 * frame))), base_view)
        ev.camera = CameraState(Camera(("perspective", 60.0, 0.1), view), LEFT, res[0] / res[1])
        for b in (cuda, orc):
            graphs[id(b)].add_to_graph(ev, res, 1, BaseRenderGraphSettings(), upload=(frame == 0))
        compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT], what=f"frame {frame}")
    # in steady state most triangles are predicted: the residual list is (much) shorter than the predicted one
    pred = cuda.readback_draw_calls(CAMERA_VIEWPORT, 0)["vertex_count"].sum()
    resid = cuda.readback_draw_calls(CAMERA_VIEWPORT, 1)["vertex_count"].sum()
    assert resid < pred


def test_config1_full_size_matches_oracle(cuda):
    """BASELINE config 1 at its full size: 10k untextured cubes, 1 directional light (2048^2 shadow map), 1920x1080 —
    the case the reference itself runs on a CPU/software adapter.  Every integer artefact identical, pixels within 1e-4."""
    from rend3_b200 import configs

    ev, res = configs.config1()
    orc = load_oracle_backend()
    settings = BaseRenderGraphSettings(clear_color=(0.10, 0.05, 0.10, 1.0))
    for b in (cuda, orc):
        BaseRenderGraph(b).add_to_graph(ev, res, 1, settings)
    compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT, 0], what="config 1")
    assert cuda.visible_count(CAMERA_VIEWPORT) > 5000


def test_config5_full_size_matches_oracle(cuda):
    """BASELINE config 5 at full size (3840x2160, ~500k triangles, 64 point + 4 shadowed directional lights), one frame:
    every integer artefact, the four shadow maps and the depth buffer bit-exact, the HDR pixels within TOL."""
    from rend3_b200 import configs

    ev, res = configs.config5()
    orc = load_oracle_backend()
    for b in (cuda, orc):
        BaseRenderGraph(b).add_to_graph(ev, res, 1, BaseRenderGraphSettings(clear_color=(0.10, 0.05, 0.10, 1.0)))
    compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT, 0, 3], what="config 5")
    st = cuda.forward_stats()
    assert st[:3] == orc.forward_stats()[:3] and st[2] == res[0] * res[1], "the slabs close the frame: every pixel is shaded"


def test_config3_full_size_matches_oracle(cuda):
    """BASELINE config 3 at full size (200k objects over 1000 meshes / 20 M triangles, 4 shadow maps + 4 point lights, 3840x2160):
    the first frame (all residual) artefact by artefact for the viewport and one shadow camera, then a second frame (predicted list,
    hi-Z occlusion at scale) through its draw records and pixels."""
    from rend3_b200 import configs

    ev, res = configs.config3()
    orc = load_oracle_backend()
    graphs = {id(b): BaseRenderGraph(b) for b in (cuda, orc)}
    settings = BaseRenderGraphSettings(clear_color=(0.10, 0.05, 0.10, 1.0))
    for b in (cuda, orc):
        graphs[id(b)].add_to_graph(ev, res, 1, settings)
    compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT, 2], what="config 3 frame 0")
    assert cuda.forward_stats()[:3] == orc.forward_stats()[:3]
    for b in (cuda, orc):
        graphs[id(b)].add_to_graph(ev, res, 1, settings, upload=False)
    for part in (0, 1):
        do = orc.readback_draw_calls(CAMERA_VIEWPORT, part)
        assert cuda.readback_draw_calls(CAMERA_VIEWPORT, part)[:len(do)].tobytes() == do.tobytes(), f"frame 1 draw calls, partition {part}"
    assert np.array_equal(cuda.readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32))
    hdr_close(cuda.readback_hdr_f32(), orc.readback_hdr_f32(), "config 3 frame 1 hdr")
    sc, so = cuda.forward_stats(), orc.forward_stats()
    assert sc[:3] == so[:3]


def test_full_size_cull_bake_properties(cuda):
    """BASELINE configs 2 / 4 at full size (10 M object records on one GPU), checked through size-independent properties:
    sortedness, agreement with an independent float64 classification away from the plane boundaries, idempotence,
    cull-only == cull+bake, and linearity of the baked matrices on a sample."""
    n = 10_000_000
    rec = object_cloud_records(n, seed=4)
    cam = cloud_camera()
    header = per_camera_header(cam, CAMERA_VIEWPORT, (1920, 1080), 1, n)
    cuda.set_objects(rec)
    cuda.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE | CB_CULL)
    vis = cuda.readback_visible(CAMERA_VIEWPORT).copy()
    assert np.all(np.diff(vis.astype(np.int64)) > 0), "ascending, no duplicates"
    fr = cam.world_frustum.astype(np.float64)
    margin = rec["sphere_center"].astype(np.float64) @ fr[:, :3].T + fr[:, 3] + rec["sphere_radius"].astype(np.float64)[:, None]
    enabled = rec["enabled"] != 0
    mask = np.zeros(n, dtype=bool)
    mask[vis] = True
    eps = 1e-2 * (1.0 + np.abs(margin))   # f32 evaluation error of a 2000-unit world
    assert mask[(margin > eps).all(axis=1) & enabled].all(), "objects clearly inside must be listed"
    assert not mask[(margin < -eps).any(axis=1) | ~enabled].any(), "objects clearly outside / disabled must not be listed"
    cuda.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE | CB_CULL)
    assert np.array_equal(cuda.readback_visible(CAMERA_VIEWPORT), vis), "idempotent"
    cuda.object_uniform_upload(CAMERA_VIEWPORT, header, CB_CULL)
    assert np.array_equal(cuda.readback_visible(CAMERA_VIEWPORT), vis), "cull-only lists the same set"
    sample = np.linspace(0, n - 1, 257).astype(np.int64)
    vp = cam.view_proj.astype(np.float64).T
    for i in sample:
        if enabled[i]:
            m = cuda.readback_object_matrices(CAMERA_VIEWPORT, int(i), 1)[0]
            t = rec["transform"][i].reshape(4, 4).astype(np.float64).T
            assert np.allclose(m["model_view_proj"].reshape(4, 4).T, vp @ t, rtol=2e-5, atol=2e-2)


def test_msaa_four_frame_matches_oracle(cuda):
    """SampleCount::Four: per-sample coverage / depth, one shade per pixel and primitive, box resolve, min-depth hi-Z;
    two frames so that the multisampled predicted + residual passes and the MULTISAMPLED cull flag are exercised."""
    res = (256, 160)
    ev = cube_field_scene(n_objects=800, seed=21, resolution=res, n_point_lights=2, shadow_resolution=256, shadow_distance=100.0, pull_back=6.0, extent=12.0,
                          subdivisions=(1, 2))
    orc = load_oracle_backend()
    graphs = {id(b): BaseRenderGraph(b) for b in (cuda, orc)}
    for frame in range(2):
        for b in (cuda, orc):
            graphs[id(b)].add_to_graph(ev, res, 4, BaseRenderGraphSettings(clear_color=(0.2, 0.1, 0.3, 1.0)), upload=(frame == 0))
        compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT, 0], what=f"msaa frame {frame}", f16_samples=True)
    assert cuda.forward_stats()[1] > cuda.forward_stats()[2] > 0


def test_near_plane_clipping_and_large_triangles(cuda):
    """Camera inside the field: triangles cross the near plane (clipper) and cover many bands (large path)."""
    res = (384, 216)
    ev = cube_field_scene(n_objects=400, seed=9, resolution=res, n_dir_lights=1, shadow_resolution=256, shadow_distance=60.0,
                          pull_back=0.6, extent=6.0)
    orc = load_oracle_backend()
    for b in (cuda, orc):
        BaseRenderGraph(b).add_to_graph(ev, res, 1, BaseRenderGraphSettings(clear_color=(0, 0, 0, 1)))
    compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT, 0], what="near-plane")
    assert cuda.forward_stats()[2] > 0.3 * res[0] * res[1]


def test_empty_and_ragged_inputs(cuda):
    res = (64, 64)
    # empty world: nothing visible, clear colour everywhere
    ev = cube_field_scene(n_objects=0, seed=1, resolution=res, n_dir_lights=0)
    BaseRenderGraph(cuda).add_to_graph(ev, res, 1, BaseRenderGraphSettings(clear_color=(0.25, 0.5, 0.75, 1.0)))
    assert cuda.visible_count(CAMERA_VIEWPORT) == 0
    assert np.allclose(cuda.readback_hdr_f32(), np.array([0.25, 0.5, 0.75, 1.0], dtype=np.float32))
    # every object disabled
    ev = cube_field_scene(n_objects=100, seed=1, resolution=res, n_dir_lights=0)
    ev.object_buffer["enabled"][:] = 0
    ev.object_live[:] = 0
    orc = load_oracle_backend()
    for b in (cuda, orc):
        BaseRenderGraph(b).add_to_graph(ev, res, 1, BaseRenderGraphSettings())
    assert cuda.visible_count(CAMERA_VIEWPORT) == 0
    assert np.array_equal(cuda.readback_ldr(), orc.readback_ldr())


# ------------------------------------------------------------------ the reference's golden scenes through the CUDA path
def test_reference_goldens_on_cuda(cuda):
    from functools import partial

    import reference_goldens as g

    load = partial(load_cuda_backend, 0)
    g.empty(load)
    for args in [("Left", "Cw", True), ("Left", "Ccw", False), ("Right", "Cw", False), ("Right", "Ccw", True)]:
        g.triangle(load, *args)
    g.coordinate_space(load)
    g.sample_coverage(load, 1)
    g.sample_coverage(load, 4)
    g.msaa_four(load)
    g.multi_frame_add(load)
    g.duplicate_object_retain(load)
    g.shadow_plane(load)
    g.shadow_cube(load)
    g.cube_example_screenshot(load)


def test_error_paths(cuda):
    from rend3_b200.backend import R3Error

    with pytest.raises(R3Error):
        cuda.set_render_target(64, 64, 2)           # SampleCount is One or Four (rend3-types SampleCount)
    with pytest.raises(R3Error):
        cuda.readback_hiz(99)
    rec = np.zeros(4, dtype=OBJECT_DTYPE)
    cuda.set_objects(rec)
    hdr = per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (64, 64), 1, 9)   # object_count > buffer
    with pytest.raises(R3Error):
        cuda.object_uniform_upload(CAMERA_VIEWPORT, hdr)
    # texture table: a mip chain that does not fit its blob, an unknown format
    from rend3_b200.layouts import TEXTURE_DESC_DTYPE
    d = np.zeros(1, dtype=TEXTURE_DESC_DTYPE)
    d["width"], d["height"], d["mip_count"], d["format"] = 8, 8, 4, 0
    with pytest.raises(R3Error):
        cuda.set_textures(d, np.zeros(8 * 8 * 4, dtype=np.uint8))          # levels 1..3 missing
    d["mip_count"], d["format"] = 1, 31                                         # past the last format: BC6H, the integer formats, anything unknown
    with pytest.raises(R3Error):
        cuda.set_textures(d, np.zeros(8 * 8 * 4, dtype=np.uint8))
    d["width"], d["height"], d["mip_count"], d["format"] = 10, 6, 3, 9           # BC3: 3x2 + 2x1 + 1x1 blocks of 16 bytes
    cuda.set_textures(d, np.zeros(9 * 16, dtype=np.uint8))
    with pytest.raises(R3Error):
        cuda.set_textures(d, np.zeros(8 * 16, dtype=np.uint8))
    # exchange: connect before create, bad rank layout, more objects than announced
    with pytest.raises(R3Error):
        cuda.exchange_connect(CAMERA_VIEWPORT, bytes(64))
    with pytest.raises(R3Error):
        cuda.exchange_create(CAMERA_VIEWPORT, 4, 4, 100)
    cuda.exchange_create(CAMERA_VIEWPORT, 1, 0, 2)
    cuda.exchange_connect(CAMERA_VIEWPORT, bytes(64))                        # a single rank: its own buffer, no peer to open
    cuda.set_objects(np.zeros(4096, dtype=OBJECT_DTYPE))
    with pytest.raises(R3Error):
        cuda.object_uniform_upload(CAMERA_VIEWPORT, per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (64, 64), 1, 4096))
    cuda.exchange_destroy(CAMERA_VIEWPORT)
    cuda.object_uniform_upload(CAMERA_VIEWPORT, per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (64, 64), 1, 4096))
    # the single-rank exchange row mirrors the visibility words
    rec = object_cloud_records(5000, seed=3)
    cuda.set_objects(rec)
    cuda.exchange_create(CAMERA_VIEWPORT, 1, 0, 5000)
    cuda.exchange_connect(CAMERA_VIEWPORT, bytes(64))
    cuda.object_uniform_upload(CAMERA_VIEWPORT, per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (1920, 1080), 1, 5000))
    import torch

    ptr, nbytes, wpr = cuda.exchange_words(CAMERA_VIEWPORT)

    class _V:
        __cuda_array_interface__ = {"shape": (wpr,), "typestr": "<i4", "data": (ptr, False), "version": 2}

    cuda.sync()
    words = torch.as_tensor(_V(), device="cuda:0").cpu().numpy().view(np.uint32)
    bits = np.unpackbits(words.view(np.uint8), bitorder="little")[:5000]
    assert np.array_equal(np.nonzero(bits)[0].astype(np.uint32), cuda.readback_visible(CAMERA_VIEWPORT))
    cuda.exchange_destroy(CAMERA_VIEWPORT)


def test_single_rank_exchange_consumers(cuda):
    """With one rank the exchange consumers must reproduce the local compaction: exchange_merge lists exactly the visible objects
    (several 32768-object tiles and a partial last word, so the tile prefix and the tail mask take part), and exchange_merge and
    exchange_count both report that count for the rank and in total."""
    import torch

    def device_u32(ptr, n):
        class View:
            __cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 2}
        return torch.as_tensor(View(), device="cuda:0").cpu().numpy().view(np.uint32)

    n = 70_001
    cuda.set_objects(object_cloud_records(n, seed=8))
    cuda.exchange_create(CAMERA_VIEWPORT, 1, 0, n)
    cuda.exchange_connect(CAMERA_VIEWPORT, bytes(64))
    cuda.object_uniform_upload(CAMERA_VIEWPORT, per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (1920, 1080), 1, n))
    vis = cuda.readback_visible(CAMERA_VIEWPORT)
    assert 0 < len(vis) < n
    cuda.exchange_merge(CAMERA_VIEWPORT, [n])
    lst, cnt, _ = cuda.exchange_merged(CAMERA_VIEWPORT)
    cuda.sync()
    n_merged = int(device_u32(cnt, 1)[0])
    assert n_merged == len(vis)
    assert np.array_equal(device_u32(lst, n_merged), vis)
    assert cuda.exchange_counts(CAMERA_VIEWPORT, 1).tolist() == [len(vis), len(vis)]
    cuda.exchange_count(CAMERA_VIEWPORT, [n])
    assert cuda.exchange_counts(CAMERA_VIEWPORT, 1).tolist() == [len(vis), len(vis)]
    cuda.exchange_destroy(CAMERA_VIEWPORT)


@pytest.mark.parametrize("far_first", [True, False])
@pytest.mark.parametrize("samples", [1, 4])
def test_blend_routine_known_answer(cuda, far_first, samples):
    """The hand-evaluated ALPHA_BLENDING chain of tests/blend_case.py (depth test + depth write, back-to-front object order)."""
    import blend_case

    r = blend_case.build(cuda, far_first)
    r.render_frame(64, samples)
    want = blend_case.expected(far_first)
    hdr = cuda.readback_hdr_f32()
    assert np.array_equal(hdr.reshape(-1, 4), np.broadcast_to(want, (64 * 64, 4))), (hdr[32, 32], want)
    assert np.allclose(cuda.readback_depth(), 0.6, rtol=0, atol=1e-6)
    assert cuda.forward_stats()[3] == 64 * 64 * samples * (2 if far_first else 1)


@pytest.mark.parametrize("samples", [1, 4])
def test_blend_routine_matches_oracle(cuda, samples):
    """Translucent cubes between opaque and cutout ones, two frames (the blend routine always draws the residual list):
    every artefact of the frame, then the blended rgba16f target within one half-precision ulp per blended layer."""
    res = (320, 180)
    ev = cube_field_scene(n_objects=1500, seed=31, resolution=res, n_dir_lights=1, n_point_lights=2, shadow_resolution=256, shadow_distance=120.0,
                          pull_back=8.0, extent=20.0, subdivisions=(1, 2), material_count=6, mixed_transparency=True, scale_range=(0.5, 2.5))
    orc = load_oracle_backend()
    graphs = {id(b): BaseRenderGraph(b) for b in (cuda, orc)}
    for frame in range(2):
        for b in (cuda, orc):
            graphs[id(b)].add_to_graph(ev, res, samples, BaseRenderGraphSettings(clear_color=(0.1, 0.2, 0.3, 1.0)), upload=(frame == 0))
        compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT, 0], check_pixels=False, what=f"blend frame {frame}")
        sc, so = cuda.forward_stats(), orc.forward_stats()
        assert so[3] > 1000 and sc[3] == so[3], (sc, so)
        assert np.array_equal(cuda.readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32)), "depth after the blend routine"
        a, o = cuda.readback_hdr_f32().astype(np.float64), orc.readback_hdr_f32().astype(np.float64)
        # every blended layer rounds to half precision: allow one f16 ulp per layer (at most 8 layers deep here) on top of TOL
        bound = TOL * np.maximum(1.0, np.abs(o)) + 8.0 * np.maximum(np.abs(o) * 2.0 ** -10, 2.0 ** -24)
        assert np.all(np.abs(a - o) <= bound), f"frame {frame}: {np.count_nonzero(np.abs(a - o) > bound)} channel values off (max {np.abs(a - o).max():.3e})"
        assert np.mean(np.abs(a - o) > TOL) < 0.02, "half-precision rounding flips must stay rare"


@pytest.mark.parametrize("sample_type", ["linear", "nearest"])
def test_texture_sampling_known_answers(cuda, sample_type):
    """textureSampleGrad (rule R9) on the CUDA path against the texture itself: level 0 at one texel per pixel, mip 1 at half
    resolution, Repeat tiling through uv_transform0, sRGB decode before filtering."""
    import texture_case as tcase
    from rend3_b200.world import Texture

    data = tcase.checker_texture(64, seed=3)
    for srgb in (False, True):
        tex = Texture(data, srgb=srgb)
        decode = tcase.srgb_decode if srgb else (lambda a: a.astype(np.float64) / 255.0)
        for size, scale, want in ((64, 1.0, decode(data)), (32, 1.0, decode(tex.levels()[1])), (128, 2.0, np.tile(decode(data), (2, 2, 1)))):
            b = load_cuda_backend(0)
            tcase.build(b, tex, sample_type, uv_scale=scale).render_frame(size)
            assert np.abs(b.readback_hdr_f32() - want).max() < 2e-5, (srgb, size, scale)
            b.close()


def test_narrow_texture_formats_known_answers(cuda):
    """R8Unorm / Rg8Unorm entries of the bindless table on the CUDA path: stored channels as unorm, missing ones (0, 0, 1)."""
    import texture_case as tcase
    from rend3_b200.world import Texture

    data = tcase.checker_texture(32, seed=5)
    for channels in (1, 2):
        b = load_cuda_backend(0)
        tcase.build(b, Texture(data, channels=channels, mips="none"), "nearest").render_frame(32)
        want = np.zeros((32, 32, 4))
        want[..., :channels] = data[..., :channels].astype(np.float64) / 255.0
        want[..., 3] = 1.0
        assert np.abs(b.readback_hdr_f32().astype(np.float64) - want).max() < 2e-6, channels
        b.close()


def test_block_compressed_formats_match_oracle_bit_for_bit():
    """BC1 - BC5 entries of the bindless table on the CUDA path (rule R11: one IEEE division of two exact integers per channel): every format
    drawn one texel per pixel — random images with punch-through BC1 blocks, both BC4 palettes, signed and sRGB variants, a size that is not
    a multiple of the block — against the float64 decode of the same blocks and, texel for texel, against the oracle."""
    import texture_case as tcase
    from rend3_b200 import bc
    from rend3_b200.world import Texture

    for size in (32, 30):
        data = tcase.checker_texture(size, seed=5)
        for name, (_, srgb_format, _) in bc.BLOCK_FORMATS.items():
            for srgb in ((False, True) if srgb_format is not None else (False,)):
                t = Texture(data, srgb=srgb, mips="none", block_format=name)
                b, orc = load_cuda_backend(0), load_oracle_backend()
                for be in (b, orc):
                    tcase.build(be, t, "nearest").render_frame(size)
                got, ref = b.readback_hdr_f32(), orc.readback_hdr_f32()
                want = bc.decode(name, t.stored_levels()[0], size, size, srgb)
                assert np.abs(got.astype(np.float64) - want).max() < 5e-7, (size, name, srgb)
                if not srgb:   # the linear formats go through no transcendental: identical bits (the sRGB curve's powf is within the pixel tolerance)
                    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), (size, name)
                else:
                    assert np.abs(got.astype(np.float64) - ref.astype(np.float64)).max() < 1e-6, (size, name)
                b.close()
    # BC7: random blocks of every mode (and the reserved one) -> the same 8-bit texels, hence the same floats, as the oracle
    blocks = tcase.random_bc7_blocks(64 * 9, seed=3).reshape(-1)
    for srgb in (False, True):
        t = Texture(np.zeros((96, 96, 4), dtype=np.uint8), srgb=srgb, mips="none", block_format="bc7", block_levels=[blocks])
        b, orc = load_cuda_backend(0), load_oracle_backend()
        for be in (b, orc):
            tcase.build(be, t, "nearest").render_frame(96)
        got, ref = b.readback_hdr_f32(), orc.readback_hdr_f32()
        assert np.abs(got.astype(np.float64) - bc.decode("bc7", blocks, 96, 96, srgb)).max() < 5e-7, srgb
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)) if not srgb else np.abs(got.astype(np.float64) - ref.astype(np.float64)).max() < 1e-6
        b.close()
    # a mip chain of blocks: levels of 8x8 .. 1x1 texels are 2x2, 1x1, 1x1, 1x1 blocks; minified 4x with the linear sampler
    data = tcase.checker_texture(32, seed=9)
    for name in ("bc1", "bc3", "bc5s", "bc7"):
        t = Texture(data, srgb=False, block_format=name)
        b, orc = load_cuda_backend(0), load_oracle_backend()
        for be in (b, orc):
            tcase.build(be, t, "linear", uv_scale=4.0).render_frame(32)
        assert np.abs(b.readback_hdr_f32().astype(np.float64) - orc.readback_hdr_f32().astype(np.float64)).max() < 1e-6, name
        b.close()


def test_ktx2_formats_match_oracle_bit_for_bit():
    """Formats 17 - 30 (snorm8, Bgra8 / sRGB, Rgb10a2, 16 / 32-bit float, unorm16) on the CUDA path: one texel per pixel against the float64
    unpack of the stored bytes and, bit for bit, against the oracle; then minified 4x through a generated mip chain with the linear sampler."""
    import texture_case as tcase
    from rend3_b200 import texformats as tf
    from rend3_b200.world import Texture

    data = tcase.checker_texture(32, seed=5)
    data[0, 0], data[0, 1] = 0, 7
    for name in tf.STORAGE:
        t = Texture(data, mips="none", storage=name)
        b, orc = load_cuda_backend(0), load_oracle_backend()
        for be in (b, orc):
            tcase.build(be, t, "nearest").render_frame(32)
        got, ref = b.readback_hdr_f32(), orc.readback_hdr_f32()
        assert np.abs(got.astype(np.float64) - tf.unpack(name, t.stored_levels()[0], 32, 32)).max() < 5e-7, name
        if name != "bgra8_srgb":
            assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), name
        b.close()
    for name in ("rgba8s", "rgb10a2", "rgba16f", "rg32f", "rgba16", "bgra8_srgb"):
        t = Texture(data, storage=name)
        b, orc = load_cuda_backend(0), load_oracle_backend()
        for be in (b, orc):
            tcase.build(be, t, "linear", uv_scale=4.0).render_frame(32)
        o = orc.readback_hdr_f32().astype(np.float64)
        assert np.abs(b.readback_hdr_f32().astype(np.float64) - o).max() < 1e-6 * max(1.0, np.abs(o).max()), name
        b.close()


@pytest.mark.parametrize("sample_type,cutout", [("linear", False), ("nearest", False), ("linear", True)])
def test_block_compressed_materials_match_oracle(cuda, sample_type, cutout):
    """The textured scene with its maps stored as BC1 / BC2 / BC3 / BC4 / BC5 / BC7 blocks (the ktx2 / dds path of rend3-gltf): every slot of
    get_pixel_data_inner reads decoded blocks, and with `cutout` the BC3 alpha decides the discard in the forward AND the shadow passes —
    depth and shadow atlas bit-identical, pixels within the tolerance."""
    from rend3_b200.scenes import textured_cube_scene

    res = (320, 180)
    ev = textured_cube_scene(n_objects=500, resolution=res, sample_type=sample_type, cutout=cutout, block_compressed=True)
    from rend3_b200.layouts import TEXFMT_BC1_RGBA_UNORM
    assert np.count_nonzero(ev.texture_descs["format"] >= TEXFMT_BC1_RGBA_UNORM) >= 7
    orc = load_oracle_backend()
    for b in (cuda, orc):
        BaseRenderGraph(b).add_to_graph(ev, res, 1, BaseRenderGraphSettings(clear_color=(0.05, 0.05, 0.1, 1.0)))
    compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT, 0], check_pixels=False, what="block compressed")
    w, h = ev.shadow_target_size
    assert np.array_equal(cuda.readback_shadow_atlas(w, h).view(np.uint32), orc.readback_shadow_atlas(w, h).view(np.uint32))
    assert np.array_equal(cuda.readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32))
    assert cuda.forward_stats()[:3] == orc.forward_stats()[:3] and orc.forward_stats()[2] > 10000
    a, o = cuda.readback_hdr_f32().astype(np.float64), orc.readback_hdr_f32().astype(np.float64)
    off = np.abs(a - o) > TOL * np.maximum(1.0, np.abs(o))
    assert not off.any(), f"{off.sum()} channel values differ (max {np.abs(a - o).max():.3e})"
    # the blocks are really sampled: the same scene with uncompressed maps gives a (slightly) different image
    plain = load_oracle_backend()
    BaseRenderGraph(plain).add_to_graph(textured_cube_scene(n_objects=500, resolution=res, sample_type=sample_type, cutout=cutout), res, 1,
                                        BaseRenderGraphSettings(clear_color=(0.05, 0.05, 0.1, 1.0)))
    assert np.abs(plain.readback_hdr_f32().astype(np.float64) - o).max() > 1e-3


@pytest.mark.parametrize("sample_type,samples", [("linear", 1), ("nearest", 1), ("linear", 4)])
def test_textured_materials_match_oracle(cuda, sample_type, samples):
    """Every texture slot and layout flag of PbrMaterial (albedo sRGB / float, tri- and bi-component normal maps, combined /
    split / bw AO-metallic-roughness, reflectance, clear coat, emissive, uv_transform0) under one shadowed directional light and
    two point lights.  Texel and mip SELECTION is bit-identical by construction for both samplers: the level comes from rule R9's
    log2_r9, a fixed sequence of IEEE operations on both sides (no libm / MUFU log2)."""
    from rend3_b200.scenes import textured_cube_scene

    res = (320, 180)
    ev = textured_cube_scene(n_objects=500, resolution=res, sample_type=sample_type)
    orc = load_oracle_backend()
    for b in (cuda, orc):
        BaseRenderGraph(b).add_to_graph(ev, res, samples, BaseRenderGraphSettings(clear_color=(0.05, 0.05, 0.1, 1.0)))
    compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT, 0], check_pixels=False, what="textured")
    assert np.array_equal(cuda.readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32))
    assert cuda.forward_stats()[:3] == orc.forward_stats()[:3] and orc.forward_stats()[2] > 10000
    a, o = cuda.readback_hdr_f32().astype(np.float64), orc.readback_hdr_f32().astype(np.float64)
    bound = TOL * np.maximum(1.0, np.abs(o)) + (np.maximum(np.abs(o) * 2.0 ** -10, 2.0 ** -24) if samples == 4 else 0.0)
    off = np.abs(a - o) > bound
    assert not off.any(), f"{off.sum()} channel values differ (max {np.abs(a - o).max():.3e})"


@pytest.mark.parametrize("samples", [1, 4])
def test_per_fragment_cutout_matches_oracle(cuda, samples):
    """Cutout materials whose alpha comes from the albedo texture and / or the vertex colour: the discard is per pixel and primitive,
    in the forward passes (opaque.wgsl:231-235) and, with depth.wgsl's own coordinates and derivatives, in the shadow pass."""
    from rend3_b200.scenes import textured_cube_scene

    res = (320, 180)
    ev = textured_cube_scene(n_objects=500, resolution=res, cutout=True)
    assert set(int(k) for k in ev.object_material_key[ev.object_live != 0]) == {0, 1}
    orc = load_oracle_backend()
    graphs = {id(b): BaseRenderGraph(b) for b in (cuda, orc)}
    for frame in range(2):
        for b in (cuda, orc):
            graphs[id(b)].add_to_graph(ev, res, samples, BaseRenderGraphSettings(clear_color=(0.05, 0.05, 0.1, 1.0)), upload=(frame == 0))
        compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT, 0], check_pixels=False, what=f"cutout frame {frame}")
        w, h = ev.shadow_target_size
        sa, so = cuda.readback_shadow_atlas(w, h).view(np.uint32), orc.readback_shadow_atlas(w, h).view(np.uint32)
        da, do = cuda.readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32)
        # the discard compares alpha with the threshold: identical arithmetic on both sides (rule R9's log2 included), so coverage is identical
        assert np.array_equal(sa, so) and np.array_equal(da, do), (np.count_nonzero(sa != so), np.count_nonzero(da != do))
        a, o = cuda.readback_hdr_f32().astype(np.float64), orc.readback_hdr_f32().astype(np.float64)
        bound = TOL * np.maximum(1.0, np.abs(o)) + (np.maximum(np.abs(o) * 2.0 ** -10, 2.0 ** -24) if samples == 4 else 0.0)
        assert not np.any(np.abs(a - o) > bound), f"{np.count_nonzero(np.abs(a - o) > bound)} channel values differ"
    # the holes are really there: the same scene without the discard covers more pixels
    opaque = load_oracle_backend()
    ev2 = textured_cube_scene(n_objects=500, resolution=res, cutout=True)
    ev2.material_buffer["alpha_cutout"] = 0.0
    BaseRenderGraph(opaque).add_to_graph(ev2, res, samples, BaseRenderGraphSettings(clear_color=(0.05, 0.05, 0.1, 1.0)))
    assert np.count_nonzero(opaque.readback_depth() > 0) > np.count_nonzero(orc.readback_depth() > 0) + 100


def test_cpp_host_mirror_renders_the_same_frames(cuda, tmp_path):
    """The native host layer (include/rend3_b200.hpp: GpuCuller / ForwardRoutine / BaseRenderGraph in base.rs order) driven by
    rend3_b200/host/r3_frame on a dumped scene: two frames, same artefacts as the Python-driven context and the oracle."""
    import subprocess

    from rend3_b200.scene_io import dump_scene, load_outputs

    res = (256, 144)
    ev = cube_field_scene(n_objects=900, seed=17, resolution=res, n_dir_lights=1, n_point_lights=2, shadow_resolution=256, shadow_distance=100.0, pull_back=7.0,
                          extent=14.0, subdivisions=(1, 2), material_count=6, mixed_transparency=True)
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.2, 0.3, 1.0))
    scene, out = tmp_path / "scene.r3s", tmp_path / "out.r3o"
    dump_scene(str(scene), ev, res, 1, settings, True, frames=2)
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rend3_b200", "host", "r3_frame")
    r = subprocess.run([exe, str(scene), str(out)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    got = load_outputs(str(out))
    # the same frames submitted as one CUDA graph each (r3::BaseRenderGraph::submit_as_graph): identical artefacts
    out_g = tmp_path / "out_graph.r3o"
    r = subprocess.run([exe, str(scene), str(out_g)], capture_output=True, text=True, timeout=300, env=dict(os.environ, R3_FRAME_GRAPH="1"))
    assert r.returncode == 0, r.stdout + r.stderr
    got_g = load_outputs(str(out_g))
    for k in got:
        assert np.array_equal(got[k], got_g[k]), f"graph submission changed `{k}`"
    orc = load_oracle_backend()
    graphs = {id(b): BaseRenderGraph(b) for b in (cuda, orc)}
    for frame in range(2):
        for b in (cuda, orc):
            graphs[id(b)].add_to_graph(ev, res, 1, settings, upload=(frame == 0))
    assert np.array_equal(got["visible"], orc.readback_visible(CAMERA_VIEWPORT))
    assert np.array_equal(got["depth"].view(np.uint32), orc.readback_depth().reshape(-1).view(np.uint32))
    assert list(got["stats"][:3]) == list(orc.forward_stats()[:3])
    assert np.array_equal(got["hdr"], cuda.readback_hdr_f32().reshape(-1)), "same library, same calls: the two host layers must agree bit for bit"
    assert np.abs(got["ldr"].astype(int) - orc.readback_ldr().reshape(-1).astype(int)).max() <= 1


def test_skybox_known_answers_and_parity(cuda):
    """SkyboxRoutine (skybox.wgsl, rule R10): the six axis views on CUDA, then a cube field with opaque, cutout and translucent objects
    in front of a random cube map, single- and multi-sampled, against the oracle."""
    import dataclasses

    import skybox_case as sk

    for f in range(6):
        b = load_cuda_backend(0)
        sk.build(b, sk.solid_faces(), f).render_frame(32)
        want = np.append(sk.FACE_COLOURS[f][:3].astype(np.float32) / 255.0, 1.0)
        assert np.array_equal(b.readback_hdr_f32().reshape(-1, 4), np.broadcast_to(want, (32 * 32, 4))), f
        b.close()
    from rend3_b200.world import Renderer

    res = (320, 180)
    ev = cube_field_scene(n_objects=400, seed=23, resolution=res, n_dir_lights=1, shadow_resolution=256, shadow_distance=100.0, pull_back=8.0, extent=14.0,
                          subdivisions=(1, 2), material_count=6, mixed_transparency=True, scale_range=(0.5, 2.0))
    rng = np.random.default_rng(9)
    sky = Renderer()
    sky.set_skybox([np.kron(rng.integers(0, 256, (8, 8, 4), dtype=np.uint8), np.ones((8, 8, 1), dtype=np.uint8)) for _ in range(6)], srgb=True)
    desc, blob = sky._skybox_blob()
    ev = dataclasses.replace(ev, skybox_desc=desc, skybox_texels=blob)
    for samples in (1, 4):
        orc, b = load_oracle_backend(), load_cuda_backend(0)
        for x in (b, orc):
            BaseRenderGraph(x).add_to_graph(ev, res, samples, BaseRenderGraphSettings(clear_color=(0.0, 0.0, 0.0, 1.0)))
        a, o = b.readback_hdr_f32().astype(np.float64), orc.readback_hdr_f32().astype(np.float64)
        assert np.count_nonzero(orc.readback_depth() == 0.0) > 5000, "the sky must be visible"
        assert np.array_equal(b.readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32))
        # translucent layers (and MSAA samples) round to rgba16f before they are compared: a few half-precision ulps on top of TOL
        bound = TOL * np.maximum(1.0, np.abs(o)) + 8.0 * np.maximum(np.abs(o) * 2.0 ** -10, 2.0 ** -24)
        assert np.all(np.abs(a - o) <= bound), f"samples {samples}: {np.count_nonzero(np.abs(a - o) > bound)} channel values off (max {np.abs(a - o).max():.3e})"
        b.close()


def test_ragged_meshes_and_batch_boundaries(cuda):
    """Edge shapes of the invocation space: meshes with 0, 1, 255, 256 and 257 triangles (none / one / exactly one / two workgroups,
    batching.rs:192,235 pads to 256), 257 objects per material so that batches fill to exactly 256 objects and regions split on key
    changes, a disabled object in the middle; two frames."""
    from rend3_b200.world import CUTOUT, LEFT, MeshBuilder, Object, PbrMaterial, Renderer

    def strip_mesh(n_tris, seed):
        # a fan of n_tris small triangles around the origin, all facing the camera (Cw in a left-handed world)
        rng = np.random.default_rng(seed)
        pos, idx = [], []
        for t in range(n_tris):
            a = 2 * np.pi * t / max(n_tris, 1)
            c = np.array([0.8 * np.cos(a), 0.8 * np.sin(a), 0.0]) * (0.3 + 0.7 * rng.random())
            base = len(pos)
            pos += [c + (0.06, -0.05, 0), c + (-0.06, -0.05, 0), c + (0, 0.07, 0)]
            idx += [base, base + 1, base + 2]
        if not pos:
            pos = [(0, 0, 0), (0, 0, 0), (0, 0, 0)]
        return MeshBuilder.new(np.array(pos, dtype=np.float32), LEFT).with_indices(np.array(idx, dtype=np.uint32)).build()

    res = (256, 256)
    r = Renderer(LEFT, aspect_ratio=1.0)
    meshes = [r.add_mesh(strip_mesh(n, 50 + n)) for n in (0, 1, 255, 256, 257)]
    # the middle material is a cutout that never discards: material key 1, so a region boundary falls inside a batch
    mats = [r.add_material(PbrMaterial(albedo_value=(0.2 + 0.2 * m, 0.5, 0.9 - 0.2 * m, 1.0), unlit=True, transparency=CUTOUT if m == 1 else 0)) for m in range(3)]
    r.set_camera_data(Camera(("perspective", 60.0, 0.1), glam.look_at_lh(np.array([0, 0, -6], dtype=np.float32), np.zeros(3, dtype=np.float32),
                                                                           np.array([0, 1, 0], dtype=np.float32))))
    rng = np.random.default_rng(77)
    handles = []
    for i in range(3 * 257):
        t = glam.mul(glam.from_translation(tuple(rng.uniform(-2.5, 2.5, 3))), glam.from_scale((0.5, 0.5, 0.5)))
        handles.append(r.add_object(Object(meshes[i % 5], mats[i // 257], t)))
    ev = r.evaluate()
    ev.object_buffer["enabled"][handles[300]] = 0
    orc = load_oracle_backend()
    graphs = {id(b): BaseRenderGraph(b) for b in (cuda, orc)}
    for frame in range(2):
        for b in (cuda, orc):
            graphs[id(b)].add_to_graph(ev, res, 1, BaseRenderGraphSettings(clear_color=(0, 0, 0, 1)), upload=(frame == 0))
        compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT], what=f"ragged frame {frame}")
    bo, ro = orc.readback_batches(CAMERA_VIEWPORT)
    assert len(bo) >= 3 and int(bo[0]["total_objects"]) == 256, "the first batch must be full"
    assert len(ro) > len(bo) and set(int(k) for k in ro["material_key"]) == {0, 1}, "a key change must split a batch into regions"
    assert orc.forward_stats()[2] > 500


def test_nan_and_signed_zero_distances_sort_like_ordered_float(cuda, monkeypatch):
    """Object locations holding NaN / inf, and objects exactly at the viewport location (distance +0.0, or -0.0 after the back-to-front
    negation): device batching, host batching and the oracle must produce the same batch tables — OrderedFloat's total order
    (NaN greatest and equal to itself, -0.0 == +0.0; batching.rs:37,156-164)."""
    res = (200, 120)
    ev = cube_field_scene(n_objects=700, seed=41, resolution=res, n_dir_lights=0, pull_back=8.0, extent=16.0, subdivisions=(1,), material_count=6,
                          mixed_transparency=True)
    rng = np.random.default_rng(3)
    live = np.nonzero(ev.object_live)[0]
    pick = rng.permutation(live)
    ev.object_location[pick[:40]] = np.nan
    ev.object_location[pick[40:60], 1] = np.inf
    ev.object_location[pick[60:120]] = np.asarray(ev.camera.location(), dtype=np.float32)   # distance exactly 0
    orc = load_oracle_backend()
    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    for b in (cuda, orc):
        BaseRenderGraph(b).add_to_graph(ev, res, 1, BaseRenderGraphSettings())
    assert cuda.batching_info(CAMERA_VIEWPORT)["path"] == "device"
    compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT], check_pixels=False, what="NaN distances, device batching")
    monkeypatch.setenv("R3_HOST_BATCHING", "1")
    host = load_cuda_backend(0)
    BaseRenderGraph(host).add_to_graph(ev, res, 1, BaseRenderGraphSettings())
    assert host.batching_info(CAMERA_VIEWPORT)["path"] == "host"
    compare_frame_state(host, orc, ev, [CAMERA_VIEWPORT], check_pixels=False, what="NaN distances, host batching")
    host.close()


def test_frames_submitted_as_cuda_graphs_match_oracle(monkeypatch):
    """r3_frame_begin / r3_frame_end: the frame is recorded by stream capture and submitted as ONE graph launch (graph.rs:510: one submit
    per frame); from the third frame on the instantiated graph of the same parity is only updated.  Five frames with a moving camera
    (new kernel arguments every frame) and translucent objects (the blend routine reads a counter back: an early flush): every artefact
    of every frame equals the oracle's, exactly as in eager submission."""
    monkeypatch.setenv("R3_FRAME_GRAPH", "1")
    from rend3_b200.world import CameraState, LEFT
    res = (320, 200)
    for mixed in (False, True):
        ev = cube_field_scene(n_objects=1500, seed=3, resolution=res, n_dir_lights=1, shadow_resolution=256, shadow_distance=100.0, pull_back=8.0, extent=20.0,
                              subdivisions=(1, 2), material_count=6 if mixed else 1, mixed_transparency=mixed)
        b, orc = load_cuda_backend(0), load_oracle_backend()
        graphs = {id(x): BaseRenderGraph(x) for x in (b, orc)}
        base_view = ev.camera.view.copy()
        for frame in range(5):
            view = glam.mul(glam.from_rotation_y(np.float32(np.radians(0.5 * frame))), base_view)
            ev.camera = CameraState(Camera(("perspective", 60.0, 0.1), view), LEFT, res[0] / res[1])
            for x in (b, orc):
                graphs[id(x)].add_to_graph(ev, res, 1, BaseRenderGraphSettings(clear_color=(0.1, 0.2, 0.3, 1.0)), upload=(frame == 0))
            compare_frame_state(b, orc, ev, [CAMERA_VIEWPORT, 0], check_pixels=not mixed, what=f"graph frame {frame} (mixed={mixed})")
            if mixed:
                assert np.array_equal(b.readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32))
        st = b.frame_graph_stats()
        assert st["frames"] == 5, st
        if not mixed:
            # the first frame allocates (early flush, the rest of it runs eagerly); from then on every frame is one graph launch, and the
            # instantiated graphs (one per ping-pong parity) are only updated
            assert st["graphed"] >= 4 and st["flushed"] <= 1 and st["instantiations"] <= 2, st
        else:
            assert st["flushed"] >= 4, st                                   # the blend routine's pool check flushes the recording every frame
        b.close()


@pytest.mark.parametrize("frame_sort", ["0", "1"])
def test_frame_wide_sort_equals_per_camera_sort(monkeypatch, frame_sort):
    """The cameras of a frame share one sort (the key does not depend on the camera, batching.rs:156-157) and take their visible
    objects out of it by stream compaction — or sort their own visible lists: both must give the oracle's batch tables, for the
    viewport and for shadow cameras, over three frames (the per-camera previous-invocation maps follow along)."""
    monkeypatch.setenv("R3_FRAME_SORT", frame_sort)
    res = (320, 180)
    ev = cube_field_scene(n_objects=9000, seed=52, resolution=res, n_dir_lights=2, shadow_resolution=256, shadow_distance=150.0, pull_back=9.0, extent=30.0,
                          subdivisions=(1, 2), material_count=6, mixed_transparency=True)
    b, orc = load_cuda_backend(0), load_oracle_backend()
    graphs = {id(x): BaseRenderGraph(x) for x in (b, orc)}
    for frame in range(3):
        for x in (b, orc):
            graphs[id(x)].add_to_graph(ev, res, 1, BaseRenderGraphSettings(), upload=(frame == 0))
        assert b.batching_info(CAMERA_VIEWPORT)["path"] == ("device, frame-wide sort" if frame_sort == "1" else "device")
        compare_frame_state(b, orc, ev, [CAMERA_VIEWPORT, 0, 1], check_pixels=(frame == 2), what=f"frame sort {frame_sort}, frame {frame}", f16_samples=True)
    b.close()


@pytest.mark.parametrize("frame_sort", ["0", "1"])
def test_device_batching_beyond_the_cooperative_sort_matches_oracle(cuda, monkeypatch, frame_sort):
    """More than 524288 sort candidates (2048-key tiles x 256 cooperative CTAs) take the multi-launch radix sort: key generation,
    then five histogram / scan / scatter launches.  Per-camera sort of the visible list (itself past that size) and frame-wide sort
    of every slot, three material keys, both sorting reasons and both orders: the batch tables equal the oracle's."""
    monkeypatch.setenv("R3_FRAME_SORT", frame_sort)
    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    n = 1_200_000
    rec = object_cloud_records(n, seed=4)
    rng = np.random.default_rng(17)
    key = rng.integers(0, 3, n).astype(np.uint64)
    flags = (1 | 2 * rng.integers(0, 2, n) | 4 * rng.integers(0, 2, n)).astype(np.uint8)   # live | atomic-capable | back to front
    header = per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (1920, 1080), 1, n)
    orc = load_oracle_backend()
    for b in (cuda, orc):
        b.set_objects(rec)
        b.set_object_sort_info(key, flags, rec["sphere_center"])
        b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_CULL)
        b.batch_objects(CAMERA_VIEWPORT, np.zeros(3, dtype=np.float32))
    assert cuda.batching_info(CAMERA_VIEWPORT)["path"] == ("device, frame-wide sort" if frame_sort == "1" else "device")
    assert orc.visible_count(CAMERA_VIEWPORT) > 2048 * 256
    bc, rc = cuda.readback_batches(CAMERA_VIEWPORT)
    bo, ro = orc.readback_batches(CAMERA_VIEWPORT)
    assert len(bc) == len(bo) and rc.tobytes() == ro.tobytes()
    for f in ("total_objects", "total_invocations", "batch_base_invocation"):
        assert np.array_equal(bc[f], bo[f]), f
    # every batch is full except the last; its slots past total_objects are unspecified (batching.rs:186)
    info_c, info_o = bc["object_culling_information"], bo["object_culling_information"]
    n_last = int(bo[-1]["total_objects"])
    assert info_c[:-1].tobytes() == info_o[:-1].tobytes()
    assert info_c[-1][:n_last].tobytes() == info_o[-1][:n_last].tobytes()


def test_device_batching_equals_host_batching_and_oracle(cuda, monkeypatch):
    """batch_objects on the device (radix sort + block scans) against the host implementation and the oracle, with
    three material keys (opaque / cutout / blend: atomic and non-atomic regions, front-to-back and back-to-front)."""
    res = (320, 180)
    ev = cube_field_scene(n_objects=3000, seed=12, resolution=res, n_dir_lights=1, shadow_resolution=256, shadow_distance=120.0, pull_back=9.0,
                          extent=25.0, subdivisions=(1, 2, 5), material_count=6, mixed_transparency=True)
    orc = load_oracle_backend()
    BaseRenderGraph(orc).add_to_graph(ev, res, 1, BaseRenderGraphSettings())
    BaseRenderGraph(cuda).add_to_graph(ev, res, 1, BaseRenderGraphSettings())
    compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT, 0], what="device batching", f16_samples=True)
    bo, ro = orc.readback_batches(CAMERA_VIEWPORT)
    assert len(bo) > 1 and len(ro) > len(bo), "scene must span several batches and split regions on key changes"
    assert set(int(r["material_key"]) for r in ro) == {0, 1, 2}
    monkeypatch.setenv("R3_HOST_BATCHING", "1")
    host = load_cuda_backend(0)
    BaseRenderGraph(host).add_to_graph(ev, res, 1, BaseRenderGraphSettings())
    compare_frame_state(host, orc, ev, [CAMERA_VIEWPORT, 0], what="host batching", f16_samples=True)
    host.close()
