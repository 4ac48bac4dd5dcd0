"""The CPU oracle's triangle cull and hi-Z pyramid against tests/cull_reference.py, a restatement of cull.wgsl and hi_z.wgsl, on scenes
aimed at the cull's edges; and the reference itself against hand-evaluated answers.  No GPU needed."""
import numpy as np
import pytest

import cull_reference as ref
import cull_scenes as scenes
import raster_scenes
from rend3_b200.backend import CAMERA_VIEWPORT
from rend3_b200.layouts import NO_PREVIOUS, PCU_MULTISAMPLED, PCU_POSITIVE_AREA_VISIBLE

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
def hiz_sizes():
    return [(1920, 1080), (3840, 2160), (40, 24), (36, 36), (34, 34), (480, 270), (481, 270), (1, 777), (777, 1), (2, 2048), (4096, 2),
            (1, 1)]


HIZ_CASES = [(w, h, 1) for w, h in hiz_sizes()] + [(1920, 1080, 4), (481, 270, 4)]
FUSED = {(1920, 1080): 3, (3840, 2160): 3, (40, 24): 3, (36, 36): 2, (34, 34): 1, (480, 270): 1, (481, 270): 0}


def hiz_content(w, h, seed):
    """Occluders for the hi-Z size tests: a far background over all but the top-left quarter and the last row and column (the uncovered
    pixels read 0), random triangles in front of it, and one-pixel quads along the whole last row and column at depths below the
    background's.  With odd sizes the unique minimum of a footprint then sits in its extra row or column.  Reverse-Z: the larger depth
    is the nearer, and the pyramid keeps the smaller.  Returns (triangles in pixels, depth per triangle)."""
    rng = np.random.default_rng(seed)
    tris, z = [], []
    x0, y0 = w // 4, h // 4
    tris += [((x0, y0), (w - 1, y0), (w - 1, h - 1)), ((x0, y0), (w - 1, h - 1), (x0, h - 1))]
    z += [0.45, 0.45]
    for _ in range(40):
        c = rng.uniform(0, 1, 2) * (w - 1, h - 1)
        t = np.clip(np.round((c + rng.uniform(-0.3, 0.3, (3, 2)) * (w, h)) * 4) / 4, 0, (w - 1, h - 1))
        tris.append(tuple(map(tuple, t)))
        z.append(float(rng.uniform(0.5, 0.9)))
    for x in range(w):
        tris += [((x, h - 1), (x + 1, h - 1), (x + 1, h)), ((x, h - 1), (x + 1, h), (x, h))]
        z += [0.05 + 0.35 * rng.random()] * 2
    for y in range(h - 1):
        tris += [((w - 1, y), (w, y), (w, y + 1)), ((w - 1, y), (w, y + 1), (w - 1, y + 1))]
        z += [0.05 + 0.35 * rng.random()] * 2
    return tris, np.array(z, F32)


def render_hiz(backend, w, h, samples, seed=0):
    tris, z = hiz_content(w, h, seed)
    r = raster_scenes.build(backend, w, h, tris, z)
    raster_scenes.draw(r, w, h, samples)
    launches = backend.launch_count()
    backend.hiz_build()
    launches = backend.launch_count() - launches
    levels = scenes.read_pyramid(backend, len(ref.hiz_dims(w, h)))
    # level 0 is the min over the samples (resolve_depth_min.wgsl:18-27), which is what the depth resolve keeps as well
    depth = backend.readback_depth()
    assert np.array_equal(levels[0].view(np.uint32), depth.view(np.uint32)), f"{w}x{h}x{samples}: level 0 is not the resolved depth"
    backend.last_hiz_launches = launches
    return levels


def assert_pyramid(levels, w, h, what):
    want = ref.hiz_pyramid(levels[0])
    assert [l.shape[::-1] for l in levels] == ref.hiz_dims(w, h), f"{what}: level sizes"
    for m in range(1, len(levels)):
        bad = levels[m].view(np.uint32) != want[m].view(np.uint32)
        assert not bad.any(), f"{what}: level {m} differs from hi_z.wgsl at {np.count_nonzero(bad)} texels, first {np.argwhere(bad)[0]}"


@pytest.mark.parametrize("w,h,samples", HIZ_CASES)
def test_oracle_hiz_matches_reference(w, h, samples):
    levels = render_hiz(load_oracle_backend(), w, h, samples)
    assert_pyramid(levels, w, h, f"oracle {w}x{h}x{samples}")
    if (w, h) in FUSED:
        assert ref.hiz_fused_levels(w, h)[0] == FUSED[(w, h)]
    assert len(np.unique(levels[0])) > 3 or w * h < 16, "the depth buffer holds too few values"
    # the last row and column hold the one-pixel quads, below everything else that was drawn
    edge = np.concatenate([levels[0][-1, :], levels[0][:, -1]])
    assert (edge > 0).all() and (edge < 0.45).all(), "the last row and column must hold the quads"


def exact_runs(backend, samples):
    """The exact decision scene under every flag combination and a shadow camera: yields (what, got, want, header)."""
    pyramid = scenes.draw_occluders(backend, samples)
    tris, z, labels = scenes.exact_decision_triangles()
    s = scenes.triangle_scene(tris, z)
    scenes.upload(backend, s)
    n = len(s.objects)
    for flags in scenes.EXACT_FLAGS:
        for cam in (CAMERA_VIEWPORT, 0):
            hdr = scenes.ortho_header(256, 256, flags, n, shadow_index=cam)
            got = scenes.run_cull(backend, s, hdr, cam)
            want = scenes.reference_for(got, s, hdr, pyramid if cam == CAMERA_VIEWPORT else None)
            yield f"flags {flags} camera {cam:#x}", s, got, want, labels, pyramid


def check_exact(what, s, got, want, labels):
    # the f32 path is exact here: float64 decides every triangle the same way
    diff = np.nonzero(want["pass32"] != want["pass64"])[0]
    assert not len(diff), f"{what}: f32 and float64 differ on {[labels[i] for i in diff[:5]]}"
    scenes.assert_matches(got, want, s, what)


@pytest.mark.parametrize("samples", [1, 4])
def test_oracle_exact_decisions_match_reference(samples):
    orc = load_oracle_backend()
    stages = set()
    for what, s, got, want, labels, pyramid in exact_runs(orc, samples):
        assert_pyramid(pyramid, 256, 256, "occluders")
        check_exact(what, s, got, want, labels)
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


def perspective_runs(backend):
    tris, labels, proj = scenes.perspective_scene()
    s = scenes.world_triangle_scene(tris)
    backend.set_render_target(64, 64, 1, (0, 0, 0, 0))
    backend.forward_begin()
    backend.hiz_build()                                   # an empty depth buffer: a uniform pyramid of 0.0
    pyramid = scenes.read_pyramid(backend, len(ref.hiz_dims(64, 64)))
    scenes.upload(backend, s)
    for flags in (0, PCU_POSITIVE_AREA_VISIBLE, PCU_MULTISAMPLED):
        hdr = scenes.ortho_header(64, 64, flags, len(s.objects), proj=proj)
        got = scenes.run_cull(backend, s, hdr)
        yield f"perspective flags {flags}", s, got, scenes.reference_for(got, s, hdr, pyramid), labels


def check_perspective(what, s, got, want, labels, margin_floor=1.0):
    """Decisions equal the f32 reference everywhere; float64 is checked where the margin allows.  Returns the excluded labels."""
    scenes.assert_matches(got, want, s, what)
    m = ref.decision_margin(want["q64"], want["stage64"], want["flags"], want["viewport"])
    near = m <= margin_floor
    bad = (want["pass32"] != want["pass64"]) & ~near
    assert not bad.any(), f"{what}: f32 and float64 differ beyond the margin on {[labels[i] for i in np.nonzero(bad)[0][:5]]}"
    unit = [i for i, l in enumerate(labels) if l == "unit w"]
    assert (want["q64"]["clip"][0][unit, 3] == 1).all(), "the unit-w triangles must have w == 1.0 exactly"
    return sorted(labels[i] for i in np.nonzero(near)[0])


def test_oracle_perspective_edges_match_reference():
    orc = load_oracle_backend()
    for what, s, got, want, labels in perspective_runs(orc):
        excluded = check_perspective(what, s, got, want, labels)
        assert len(excluded) < 30, f"{what}: {len(excluded)} margin exclusions: {excluded}"
        assert {ref.BACKFACE, ref.PASS} <= set(want["stage"][want["invocations"]].tolist())


def structural_runs(backend):
    """Yields (what, scene, got, want, census): the ragged scene over two frames (NO_PREVIOUS, then in range / past the partition),
    superblock-boundary scenes of 4 x 32768 + {-256, 0, 256} invocations, the mesh-end scene in a fresh context and again after a
    larger mesh left stale words behind the smaller one."""
    s = scenes.ragged_scene()
    scenes.upload(backend, s)
    n = len(s.objects)
    hdr = scenes.ortho_header(256, 256, 0, n)
    got = scenes.run_cull(backend, s, hdr)
    yield "ragged frame 0", s, got, scenes.reference_for(got, s, hdr, None)
    first = {}
    for b in s.batches:
        for info in b["object_culling_information"][:int(b["total_objects"])]:
            first[int(info["object_id"])] = int(b["batch_base_invocation"]) + int(info["invocation_start"])
    total = scenes.total_invocations(s.batches)
    prev = [NO_PREVIOUS if i % 3 == 0 else (first[i] if i % 3 == 1 else total + 4096 * 32 + i) for i in range(n)]
    counts = [int(c) // 3 for c in s.objects["index_count"]]
    atomic = [0 if i in (0, 1, 254, 255) else 1 for i in range(n)]
    keys = [2 if i in (0, 1, 254, 255) else 0 for i in range(n)]
    b2, r2 = scenes.build_tables(counts, atomic=atomic, keys=keys, prev=prev)
    s2 = scenes.Scene(s.objects, s.mesh, b2, r2)
    got = scenes.run_cull(backend, s2, hdr)
    yield "ragged frame 1", s2, got, scenes.reference_for(got, s2, hdr, None)
    for delta in (0, -256, 256):
        s = scenes.superblock_scene(delta)
        scenes.upload(backend, s)
        hdr = scenes.ortho_header(256, 256, PCU_POSITIVE_AREA_VISIBLE, len(s.objects))
        got = scenes.run_cull(backend, s, hdr)
        yield f"superblock {delta:+d}", s, got, scenes.reference_for(got, s, hdr, None)


def mesh_end_runs(make_backend):
    """The mesh-end scene in a fresh context, and again after a larger mesh buffer whose words past the smaller one's end are stale
    (the allocation is kept, so the bulk copy of the index runs reads them).  Closes the contexts it makes."""
    s, end, stale = scenes.mesh_end_scene()
    for with_stale in (False, True):
        b = make_backend()
        try:
            if with_stale:
                b.set_mesh_buffer(stale)
            scenes.upload(b, s)
            hdr = scenes.ortho_header(256, 256, PCU_MULTISAMPLED, len(s.objects))
            got = scenes.run_cull(b, s, hdr)
            yield f"mesh end stale={with_stale}", s, got, scenes.reference_for(got, s, hdr, None)
        finally:
            b.close()


def stale_triangles(s, stale, got, hdr):
    """The decisions of object 2's triangle 37 and object 3's first triangle when robust access is honoured, and when the stale words
    past mesh_words were read instead."""
    robust = scenes.reference_for(got, s, hdr, None)
    stale_view = scenes.Scene(s.objects, stale, s.batches, s.regions)
    wrong = scenes.reference_for(got, stale_view, hdr, None)
    picks = []
    for b in s.batches:
        for info in b["object_culling_information"][:int(b["total_objects"])]:
            g = int(b["batch_base_invocation"]) + int(info["invocation_start"])
            if int(info["object_id"]) == 2:
                picks.append(g + 37)
            if int(info["object_id"]) == 3:
                picks.append(g)
    return robust["stage"][picks], wrong["stage"][picks]


def test_oracle_structural_scenes_match_reference():
    orc = load_oracle_backend()
    for what, s, got, want in structural_runs(orc):
        scenes.assert_matches(got, want, s, what)
        assert want["pass32"].any() and not want["pass32"].all(), what
    for what, s, got, want in mesh_end_runs(load_oracle_backend):
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
    robust, wrong = stale_triangles(s, stale, got, hdr)
    assert robust.tolist() == [ref.PASS, ref.PASS] and wrong.tolist() == [ref.BACKFACE, ref.BACKFACE], (robust, wrong)


def pingpong_runs(backend):
    """The three frames of scenes.pingpong_frames, each compared as it comes (no second cull): yields (what, scene, got, want)."""
    s, frames = scenes.pingpong_frames()
    scenes.upload(backend, s)
    hdr = scenes.ortho_header(256, 256, 0, len(s.objects))
    for k, (b, r) in enumerate(frames):
        fs = scenes.Scene(s.objects, s.mesh, b, r)
        got = scenes.run_cull(backend, fs, hdr, settle=False)
        yield f"ping-pong frame {k}", fs, got, scenes.reference_for(got, fs, hdr, None)


def pingpong_census(frames):
    """The index buffer is reallocated for frame 1 (next_pow2 of its elements grows) and frame 1 and 2 read previous bits in range."""
    inv = [scenes.total_invocations(b) for b, _ in frames]
    pow2 = lambda v: 1 << (int(v) - 1).bit_length()
    assert inv[0] < inv[1] > inv[2] and pow2(3 * inv[1]) > pow2(3 * inv[0])
    for b, _ in frames[1:]:
        prev = [int(i["previous_global_invocation"]) for bb in b for i in bb["object_culling_information"][:int(bb["total_objects"])]]
        assert sum(p != NO_PREVIOUS for p in prev) >= 20


def test_oracle_pingpong_frames_match_reference():
    pingpong_census(scenes.pingpong_frames()[1])
    for what, s, got, want in pingpong_runs(load_oracle_backend()):
        scenes.assert_matches(got, want, s, what)
        if what != "ping-pong frame 0":
            resid = want["dc_resid"]["vertex_count"].sum()
            assert 0 < resid < want["dc_pred"]["vertex_count"].sum(), f"{what}: some triangles must be residual and some not"


def high_id_run(backend):
    s = scenes.high_vertex_id_scene()
    scenes.upload(backend, s)
    hdr = scenes.ortho_header(256, 256, PCU_MULTISAMPLED, len(s.objects))
    got = scenes.run_cull(backend, s, hdr)
    return s, got, scenes.reference_for(got, s, hdr, None), hdr


def check_high_id(s, got, want, hdr, what):
    scenes.assert_matches(got, want, s, what)
    assert want["pass32"].all(), f"{what}: the triangles behind ids >= 2^24 face the camera"
    masked = s.mesh.copy()
    masked[64:70] &= 0xFFFFFF
    low = scenes.reference_for(got, scenes.Scene(s.objects, masked, s.batches, s.regions), hdr, None)
    assert not low["pass32"].any(), "fetching the positions through the masked ids must decide differently"
    assert want["idx_pred"][:6].tolist() == [0, 1, 2, (1 << 24) | 0, (1 << 24) | 1, (1 << 24) | 2]
    assert want["idx_resid"][3 * 512:3 * 512 + 3].tolist() == [(2 << 24) | 3, (2 << 24) | 4, (2 << 24) | 5]


def test_oracle_high_vertex_ids_match_reference():
    orc = load_oracle_backend()
    try:
        s, got, want, hdr = high_id_run(orc)
        check_high_id(s, got, want, hdr, "oracle, ids >= 2^24")
    finally:
        orc.close()


def big_census(s, ends):
    """More than two passes of the persistent grid (4224 workgroups at 4 CTAs / SM, 5280 at 5), and the end-of-buffer objects lie in
    workgroups past the first pass, on both sides of the staging guard."""
    total = scenes.total_invocations(s.batches)
    assert total // 256 > 2 * scenes.WARP_STRIDE
    end = len(s.mesh)
    wgs = {}
    for b in s.batches:
        for info in b["object_culling_information"][:int(b["total_objects"])]:
            wgs[int(info["object_id"])] = (int(b["batch_base_invocation"]) + int(info["invocation_start"])) // 256
    assert min(wgs[o] for o in ends) > 132 * 5 * 8
    runs = [(int(s.objects[o]["first_index"]) & ~3) + 100 for o in ends]
    assert (end + 4) in runs and any(r > end + 4 for r in runs) and any(r < end + 4 for r in runs)


def test_oracle_big_scene_matches_reference():
    s, ends = scenes.big_scene()
    big_census(s, ends)
    orc = load_oracle_backend()
    scenes.upload(orc, s)
    hdr = scenes.ortho_header(256, 256, 0, len(s.objects))
    got = scenes.run_cull(orc, s, hdr)
    want = scenes.reference_for(got, s, hdr, None)
    scenes.assert_matches(got, want, s, "2.5 M invocations")
    assert want["pass32"].any() and not want["pass32"].all()


def batched_frame_runs(backend):
    """One whole frame of a small cube field through BaseRenderGraph (the batch tables from batch_objects, host- or device-built),
    then each camera's cull compared with the reference fed the tables, MVPs and pyramid that cull used."""
    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings, per_camera_header
    from rend3_b200.scenes import cube_field_scene
    res = (480, 270)
    ev = cube_field_scene(n_objects=1500, seed=5, resolution=res, n_point_lights=0, shadow_resolution=256, pull_back=12.0, extent=30.0)
    BaseRenderGraph(backend).add_to_graph(ev, res, 1, BaseRenderGraphSettings())
    pyramid = scenes.read_pyramid(backend, len(ref.hiz_dims(*res)))
    n = len(ev.object_buffer)
    cams = [(CAMERA_VIEWPORT, per_camera_header(ev.camera, CAMERA_VIEWPORT, res, 1, n), pyramid)]
    cams += [(i, per_camera_header(sh.camera, i, (sh.size, sh.size), 1, n), None) for i, sh in enumerate(ev.shadows)]
    for cam, hdr, pyr in cams:
        batches, regions = backend.readback_batches(cam)
        s = scenes.Scene(ev.object_buffer, np.asarray(ev.mesh_buffer, np.uint32), batches, regions)
        got = dict(words=backend.readback_culling_results(cam, 0), prev=backend.readback_culling_results(cam, 1),
                   dc_pred=backend.readback_draw_calls(cam, 0), dc_resid=backend.readback_draw_calls(cam, 1),
                   idx_pred=backend.readback_indices(cam, 0), idx_resid=backend.readback_indices(cam, 1),
                   mvps=backend.readback_object_matrices(cam, 0, n)["model_view_proj"].reshape(n, 16))
        yield f"frame camera {cam:#x}", s, got, scenes.reference_for(got, s, hdr, pyr)


def test_oracle_host_batched_frame_matches_reference():
    stages = set()
    for what, s, got, want in batched_frame_runs(load_oracle_backend()):
        scenes.assert_matches(got, want, s, what)
        stages |= set(want["stage"][want["invocations"]].tolist())
    assert {ref.BACKFACE, ref.PASS} <= stages
