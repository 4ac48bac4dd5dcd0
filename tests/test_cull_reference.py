"""The CPU oracle's triangle cull and hi-Z pyramid against tests/cull_reference.py, a restatement of cull.wgsl and hi_z.wgsl, on scenes
aimed at the cull's edges; and the reference itself against hand-evaluated answers.  No GPU needed."""
import numpy as np
import pytest

import cull_reference as ref
import cull_scenes as scenes
from rend3_b200.layouts import PCU_MULTISAMPLED, PCU_POSITIVE_AREA_VISIBLE

from oracle import load_oracle_backend

F32 = np.float32
ORTHO = scenes.ortho_header(256, 256, 0, 1)["view_proj"].reshape(1, 16)


def one(tri_px, flags=0, z=0.5, pyramid=None, viewport=True):
    t = np.zeros((1, 3, 3), F32)
    t[0, :, :2] = tri_px
    t[0, :, 2] = z
    p, stage, q = ref.execute_culling(ORTHO, t, flags, (256, 256), viewport, pyramid)
    return bool(p[0]), int(stage[0]), q


# ------------------------------------------------------------------ hand-evaluated answers
def test_ceil_log2_known_answers():
    x = np.array([0.5, 1.0, np.nextafter(F32(1), F32(2)), 2.0, 3.0, 4.0, np.nextafter(F32(4), F32(5)), 2.0 ** 100, np.inf, np.nan], F32)
    assert ref.ceil_log2(x).tolist() == [0, 0, 1, 1, 2, 2, 3, 100, 128, 0]
    assert ref.ceil_log2_f64(x.astype(np.float64)).tolist() == [0, 0, 1, 1, 2, 2, 3, 100, 128, 0]


def test_pixel_centre_ties_round_to_even():
    """A screen box [x + 0.5, x + 1.5]: round() ties to even, so for even x the ends round to x and x + 2 (a centre is inside), for odd
    x both round to x + 1 (culled).  Half away from zero would keep both."""
    for x, keep in ((40, True), (41, False), (170, True), (171, False)):
        box = ((x + 0.5, 60), (x + 1.5, 60), (x + 0.5, 80))
        for flip in (False, True):
            t = np.array(box)[:, ::-1] if flip else np.array(box)
            for tri in (t, t[[0, 2, 1]]):
                p, stage, _ = one(tri, PCU_POSITIVE_AREA_VISIBLE)
                q, stage_n, _ = one(tri, 0)
                decided = [s for s in (stage, stage_n) if s != ref.BACKFACE]
                assert len(decided) == 1 and (decided[0] == ref.PASS) == keep, (x, flip, stage, stage_n)
                # multisampled targets skip the test
                assert not {one(tri, f)[1] for f in (PCU_MULTISAMPLED, PCU_MULTISAMPLED | PCU_POSITIVE_AREA_VISIBLE)} & {ref.PIXEL_CENTRE}


def test_footprint_clamps_and_strict_occlusion():
    """textureSampleMin on a 4x4 level: uv * res - 0.5 on an integer loads one texel, between integers the 2x2 around it; outside
    [0, 1] and at a NaN coordinate the texels clamp.  The mip clamps to the last level; the occlusion test is strict."""
    lvl = np.arange(16, dtype=F32).reshape(4, 4) + 1
    pyr = [lvl, np.array([[0.5, 0.25], [0.75, 1.0]], F32), np.array([[0.125]], F32)]
    s = lambda u, v, m: float(ref.texture_sample_min(pyr, np.array([u], F32), np.array([v], F32), np.array([m]))[0])
    assert s(0.375, 0.375, 0) == lvl[1, 1]                  # 0.375 * 4 - 0.5 = 1: one texel
    assert s(0.5, 0.5, 0) == lvl[1, 1]                      # 1.5: texels 1 and 2 on both axes, the min is (1, 1)
    assert s(0.5625, 0.9, 0) == lvl[3, 1]                   # x 1.75 -> 1, 2; y 3.1 -> 3 and ceil 4 clamped to 3
    assert s(-3.0, 0.125, 0) == lvl[0, 0]                   # far left: both x texels clamp to 0
    assert s(7.0, 7.0, 0) == lvl[3, 3]
    assert s(0.75, 0.25, 1) == 0.25 and s(0.5, 0.5, 1) == 0.25
    assert s(0.9, 0.9, 9) == 0.125                          # mip past the chain: the last level
    # the triangle faces the camera under PCU_POSITIVE_AREA_VISIBLE; the test is strict: equal depth passes, one ulp behind is occluded
    flat = [np.full((256, 256), 0.5, F32)]
    front = ((20, 20), (20, 28), (28, 20))
    assert one(front, PCU_MULTISAMPLED | PCU_POSITIVE_AREA_VISIBLE, z=0.5, pyramid=flat)[1] == ref.PASS
    assert one(front, PCU_MULTISAMPLED | PCU_POSITIVE_AREA_VISIBLE, z=np.nextafter(F32(0.5), F32(0)), pyramid=flat)[1] == ref.OCCLUDED


def test_nan_coordinate_reads_the_low_and_the_high_texel():
    """A NaN uv: the low texel is max(NaN, 0) = 0, the high one min(NaN, res - 1) = res - 1; here texel res - 1 holds the minimum."""
    lvl = np.array([[0.6, 0.7, 0.8, 0.1], [0.6, 0.7, 0.8, 0.9], [0.6, 0.7, 0.8, 0.9], [0.6, 0.7, 0.8, 0.2]], F32)
    s = lambda u, v: float(ref.texture_sample_min([lvl], np.array([u], F32), np.array([v], F32), np.array([0]))[0])
    assert s(np.nan, 0.125) == F32(0.1)          # rows 0 (low, from v) and 0 (high); columns 0 and 3
    assert s(np.nan, np.nan) == F32(0.1)         # rows 0 and 3, columns 0 and 3: (0, 3) = 0.1
    assert s(0.125, np.nan) == F32(0.6)          # columns 0 and 0, rows 0 and 3


def test_hiz_pyramid_known_answers():
    """3x3 -> 1x1: the odd source folds its third row and column into the one texel; 5x2 -> 2x1 -> 1x1."""
    d = np.array([[0.9, 0.8, 0.7], [0.6, 0.5, 0.4], [0.3, 0.2, 0.1]], F32)
    p = ref.hiz_pyramid(d)
    assert [l.shape for l in p] == [(3, 3), (1, 1)] and p[1][0, 0] == F32(0.1)
    d = np.array([[0.5, 0.4, 0.3, 0.2, 0.1], [0.6, 0.7, 0.8, 0.9, 0.05]], F32)
    p = ref.hiz_pyramid(d)
    assert [l.shape for l in p] == [(2, 5), (1, 2), (1, 1)]
    # every texel of an odd-width source reads three columns: texel 0 reads x 0-2, texel 1 x 2-4
    assert p[1].tolist() == [[F32(0.3), F32(0.05)]] and p[2][0, 0] == F32(0.05)
    assert ref.hiz_pyramid(np.full((1, 1), 2.0, F32))[0][0, 0] == 2.0 and ref.hiz_pyramid(np.full((2, 2), 2.0, F32))[1][0, 0] == 1.0
    assert ref.hiz_fused_levels(1920, 1080) == (3, 1, True) and ref.hiz_fused_levels(481, 270) == (0, 2, True)


def test_packed_index_order():
    """Survivors land in ascending invocation order at their region's base, packed as batch-local object << 24 | index & 0xFFFFFF; a
    non-atomic object keeps its slots, INVALID where culled and in its padding."""
    tris = np.array([[(10, 10), (20, 10), (10, 20)]] * 3, np.float64)
    s = scenes.triangle_scene(tris, [0.5] * 3)
    hdr = scenes.ortho_header(256, 256, 0, 3)
    mvps = np.repeat(hdr["view_proj"].reshape(1, 16), 3, 0)
    batches, regions = scenes.build_tables([1, 1, 1], atomic=[1, 1, 0], keys=[0, 0, 1])
    want = ref.cull_lists(batches, regions, s.mesh, s.objects, mvps, hdr, None, np.zeros(0, np.uint32))
    assert want["pass32"].all()
    assert want["dc_pred"]["base_index"].tolist() == [0, 3 * 512] and want["dc_pred"]["vertex_count"].tolist() == [6, 0]
    assert want["dc_resid"]["vertex_count"].tolist() == [6, 3 * 256]
    assert want["idx_pred"][:6].tolist() == [0, 1, 2, (1 << 24) | 3, (1 << 24) | 4, (1 << 24) | 5]
    slot = want["idx_resid"][3 * 512:3 * 768]
    assert slot[:3].tolist() == [(2 << 24) | 6, (2 << 24) | 7, (2 << 24) | 8] and (slot[3:] == 0x00FFFFFF).all()


# ------------------------------------------------------------------ the oracle against the reference
@pytest.mark.parametrize("w,h,samples", scenes.HIZ_CASES)
def test_oracle_hiz_matches_reference(w, h, samples):
    levels = scenes.render_hiz(load_oracle_backend(), w, h, samples)
    scenes.assert_pyramid(levels, w, h, f"oracle {w}x{h}x{samples}")
    if (w, h) in scenes.FUSED:
        assert ref.hiz_fused_levels(w, h)[0] == scenes.FUSED[(w, h)]
    assert len(np.unique(levels[0])) > 3 or w * h < 16, "the depth buffer holds too few values"
    # the last row and column hold the one-pixel quads, below everything else that was drawn
    edge = np.concatenate([levels[0][-1, :], levels[0][:, -1]])
    assert (edge > 0).all() and (edge < 0.45).all(), "the last row and column must hold the quads"


@pytest.mark.parametrize("samples", [1, 4])
def test_oracle_exact_decisions_match_reference(samples):
    orc = load_oracle_backend()
    stages = set()
    for what, s, got, want, labels, pyramid in scenes.exact_runs(orc, samples):
        scenes.assert_pyramid(pyramid, 256, 256, "occluders")
        scenes.check_exact(what, s, got, want, labels)
        st = want["stage"][want["invocations"]]
        stages |= set(st.tolist())
        lab = {l: i for i, l in enumerate(labels)}
        if "camera 0xffffffff" in what and want["flags"] & PCU_MULTISAMPLED:
            # the known answers: equal depth passes, one ulp behind is occluded, and the mip at 2^k against 2^k + 1/256 decides
            for zz in (0.5, 0.25):
                a, b = st[lab[f"depth equal {zz}"]], st[lab[f"depth equal {zz} mirrored"]]
                assert ref.PASS in (a, b) and ref.BACKFACE in (a, b)
                a, b = st[lab[f"depth ulp below {zz}"]], st[lab[f"depth ulp below {zz} mirrored"]]
                assert ref.OCCLUDED in (a, b)
            flips = sum(max(st[lab[f"edge 2^k k={k}"]], st[lab[f"edge 2^k k={k} mirrored"]])
                        != max(st[lab[f"edge 2^k+ k={k}"]], st[lab[f"edge 2^k+ k={k} mirrored"]]) for k in range(8))
            assert flips >= 2, "the mip boundary at 2^k must decide some triangles"
            a = max(st[lab["uv straddles A|C"]], st[lab["uv straddles A|C mirrored"]])
            assert a == ref.PASS, "a footprint straddling into the uncovered region reads its 0"
    assert stages == {ref.BACKFACE, ref.PIXEL_CENTRE, ref.OCCLUDED, ref.PASS}, stages


def test_oracle_perspective_edges_match_reference():
    orc = load_oracle_backend()
    for what, s, got, want, labels in scenes.perspective_runs(orc):
        excluded = scenes.check_perspective(what, s, got, want, labels)
        assert len(excluded) < 30, f"{what}: {len(excluded)} margin exclusions: {excluded}"
        assert {ref.BACKFACE, ref.PASS} <= set(want["stage"][want["invocations"]].tolist())


def test_oracle_structural_scenes_match_reference():
    orc = load_oracle_backend()
    for what, s, got, want in scenes.structural_runs(orc):
        scenes.assert_matches(got, want, s, what)
        assert want["pass32"].any() and not want["pass32"].all(), what
    for what, s, got, want in scenes.mesh_end_runs(load_oracle_backend):
        scenes.assert_matches(got, want, s, what)
        assert want["pass32"][:2].all(), f"{what}: the triangles at the end of the allocation must survive to be compared"


def test_mesh_end_scene_reaches_the_guard_and_the_robust_reads():
    """Object 0's staged run ends exactly at the allocation (mesh_words + 4), object 1's would end four words past it; object 2's
    indices and one of object 3's positions lie past mesh_words, and reading the stale words there instead of 0 flips both decisions."""
    s, end, stale = scenes.mesh_end_scene()
    cap = max(16, end + 4)
    starts = [int(f) & ~3 for f in s.objects["first_index"][:2]]
    assert starts[0] + 100 == cap and starts[1] + 100 == cap + 4
    assert int(s.objects["first_index"][2]) + 120 > end
    hdr = scenes.ortho_header(256, 256, PCU_MULTISAMPLED, len(s.objects))
    got = {"mvps": np.repeat(hdr["view_proj"].reshape(1, 16), 4, 0), "prev": np.zeros(0, np.uint32)}
    robust, wrong = scenes.stale_triangles(s, stale, got, hdr)
    assert robust.tolist() == [ref.PASS, ref.PASS] and wrong.tolist() == [ref.BACKFACE, ref.BACKFACE], (robust, wrong)


def test_oracle_pingpong_frames_match_reference():
    scenes.pingpong_census(scenes.pingpong_frames()[1])
    for what, s, got, want in scenes.pingpong_runs(load_oracle_backend()):
        scenes.assert_matches(got, want, s, what)
        if what != "ping-pong frame 0":
            resid = want["dc_resid"]["vertex_count"].sum()
            assert 0 < resid < want["dc_pred"]["vertex_count"].sum(), f"{what}: some triangles must be residual and some not"


def test_oracle_high_vertex_ids_match_reference():
    orc = load_oracle_backend()
    try:
        s, got, want, hdr = scenes.high_id_run(orc)
        scenes.check_high_id(s, got, want, hdr, "oracle, ids >= 2^24")
    finally:
        orc.close()


def test_oracle_big_scene_matches_reference():
    s, ends = scenes.big_scene()
    scenes.big_census(s, ends)
    orc = load_oracle_backend()
    scenes.upload(orc, s)
    hdr = scenes.ortho_header(256, 256, 0, len(s.objects))
    got = scenes.run_cull(orc, s, hdr)
    want = scenes.reference_for(got, s, hdr, None)
    scenes.assert_matches(got, want, s, "2.5 M invocations")
    assert want["pass32"].any() and not want["pass32"].all()


def test_oracle_host_batched_frame_matches_reference():
    stages = set()
    for what, s, got, want in scenes.batched_frame_runs(load_oracle_backend()):
        scenes.assert_matches(got, want, s, what)
        stages |= set(want["stage"][want["invocations"]].tolist())
    assert {ref.BACKFACE, ref.PASS} <= stages
