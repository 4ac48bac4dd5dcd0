"""The CUDA triangle cull (rend3_b200/csrc/r3_tri_cull.cu) and hi-Z build (r3_shade.cu) against tests/cull_reference.py and the CPU
oracle, on the scenes of tests/cull_scenes.py: visibility words, both draw-call arrays and their zeroed tail, the defined parts of
both index lists including the non-atomic in-place slots, and every hi-Z level.  Integer artefacts: identical, not close."""
import os
import subprocess
import sys

import numpy as np
import pytest

import cull_reference as ref
import cull_scenes as scenes
from rend3_b200.backend import load_cuda_backend

from oracle import load_oracle_backend

pytestmark = pytest.mark.gpu


@pytest.fixture()
def cuda():
    b = load_cuda_backend(0)
    yield b
    b.close()


def assert_same(got, have, what):
    """Two backends' readbacks of one cull: the same words, draw calls and index lists (the CUDA buffers may be longer)."""
    for k in ("words", "dc_pred", "dc_resid"):
        n = len(have[k])
        assert got[k][:n].tobytes() == have[k].tobytes(), f"{what}: {k} differs from the oracle"
    assert np.array_equal(got["mvps"].view(np.uint32), have["mvps"].view(np.uint32)), f"{what}: baked MVPs differ from the oracle"


@pytest.mark.parametrize("w,h,samples", scenes.HIZ_CASES)
def test_hiz_levels_match_reference_and_oracle(cuda, w, h, samples):
    fused, down, tail = ref.hiz_fused_levels(w, h)
    if (w, h) in scenes.FUSED:
        assert fused == scenes.FUSED[(w, h)]
    if (w, h) == (1920, 1080):
        assert down >= 1 and tail
    if (w, h) == (3840, 2160):
        assert down == 2 and tail
    levels = scenes.render_hiz(cuda, w, h, samples)
    # what ran: the head kernel, one downsample launch per large level, the tail kernel if levels are left (r3_hiz_build)
    assert cuda.last_hiz_launches == 1 + down + int(tail), (cuda.last_hiz_launches, fused, down, tail)
    scenes.assert_pyramid(levels, w, h, f"cuda {w}x{h}x{samples}")
    orc = scenes.render_hiz(load_oracle_backend(), w, h, samples)
    for m, (a, b) in enumerate(zip(levels, orc)):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{w}x{h}x{samples}: level {m} differs from the oracle"


@pytest.mark.parametrize("samples", [1, 4])
def test_exact_decisions(cuda, samples):
    orc = {what: (got, want) for what, _, got, want, _, _ in scenes.exact_runs(load_oracle_backend(), samples)}
    stages = set()
    for what, s, got, want, labels, pyramid in scenes.exact_runs(cuda, samples):
        scenes.assert_pyramid(pyramid, 256, 256, "occluders")
        scenes.check_exact(what, s, got, want, labels)
        assert_same(got, orc[what][0], what)
        stages |= set(want["stage"][want["invocations"]].tolist())
    assert stages == {ref.BACKFACE, ref.PIXEL_CENTRE, ref.OCCLUDED, ref.PASS}, stages


def test_perspective_edges(cuda):
    orc = {what: got for what, _, got, _, _ in scenes.perspective_runs(load_oracle_backend())}
    report = []
    for what, s, got, want, labels in scenes.perspective_runs(cuda):
        excluded = scenes.check_perspective(what, s, got, want, labels)
        assert_same(got, orc[what], what)
        report.append(f"{what}: {len(excluded)} of {len(labels)} excluded from the float64 check")
        assert len(excluded) < len(labels) // 4, report[-1]
    print("\n".join(report))


def test_structural_scenes(cuda):
    orc = {what: got for what, _, got, _ in scenes.structural_runs(load_oracle_backend())}
    for what, s, got, want in scenes.structural_runs(cuda):
        scenes.assert_matches(got, want, s, what)
        assert_same(got, orc[what], what)
        if what == "ragged frame 1":
            resid = want["dc_resid"]["vertex_count"][scenes.regions_atomic(s)].sum()
            pred = want["dc_pred"]["vertex_count"].sum()
            assert 0 < resid < pred, "frame 1 must list some residual triangles and skip others"
        if what.startswith("superblock"):
            first = [int(b["batch_base_invocation"]) + int(i["invocation_start"]) for b in s.batches
                     for i in b["object_culling_information"][:int(b["total_objects"])]]
            assert first == [0, scenes.SB_INVOCATIONS, 3 * scenes.SB_INVOCATIONS // 2, 5 * scenes.SB_INVOCATIONS // 2], first
    for what, s, got, want in scenes.mesh_end_runs(lambda: load_cuda_backend(0)):
        scenes.assert_matches(got, want, s, what)
        assert want["pass32"][:2].all(), f"{what}: the triangles at the end of the allocation must survive to be compared"
    for what, s, got, want in scenes.pingpong_runs(cuda):
        scenes.assert_matches(got, want, s, what)


def test_high_vertex_ids(cuda):
    s, got, want, hdr = scenes.high_id_run(cuda)
    scenes.check_high_id(s, got, want, hdr, "cuda, ids >= 2^24")


@pytest.mark.parametrize("host", [False, True])
def test_batched_frame(cuda, monkeypatch, host):
    """A whole frame with batch tables from batch_objects: device batching (an upper-bound invocation total and a device-built
    header) or host batching (R3_HOST_BATCHING, read when the sort info is set), each camera's cull against the reference."""
    if host:
        monkeypatch.setenv("R3_HOST_BATCHING", "1")
    else:
        monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    for what, s, got, want in scenes.batched_frame_runs(cuda):
        scenes.assert_matches(got, want, s, what)
    assert cuda.batching_info(0xFFFFFFFF)["path"].startswith("host" if host else "device"), cuda.batching_info(0xFFFFFFFF)


def test_big_scene(cuda):
    s, ends = scenes.big_scene()
    scenes.big_census(s, ends)
    hdr = scenes.ortho_header(256, 256, 0, len(s.objects))
    scenes.upload(cuda, s)
    got = scenes.run_cull(cuda, s, hdr)
    want = scenes.reference_for(got, s, hdr, None)
    scenes.assert_matches(got, want, s, "2.5 M invocations")
    orc = load_oracle_backend()
    scenes.upload(orc, s)
    assert_same(got, scenes.run_cull(orc, s, hdr), "2.5 M invocations")


@pytest.mark.skipif(os.environ.get("R3_TEST_CTAS") == "5", reason="this is the test that runs the others with R3_TEST_CTAS=5")
def test_five_cta_variant():
    """triangle_test_kernel<5> (48 registers, 5 CTAs / SM) is chosen once per process from R3_TEST_CTAS: a subprocess runs the
    structural scenes, the 2.5 M scene and the high vertex ids with it."""
    env = dict(os.environ, R3_TEST_CTAS="5")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        "-k", "structural_scenes or big_scene or high_vertex_ids"], env=env, capture_output=True, text=True,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))), timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "3 passed" in r.stdout, r.stdout[-2000:]
