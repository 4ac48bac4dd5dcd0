"""Each raster path of rend3_b200/csrc/r3_raster.cu against the CPU oracle, bit for bit, and, where the geometry snaps exactly,
against the exact coverage reference (tests/raster_reference.py).

The set-up kernel picks a path per sub-triangle: inline by one thread (pixel box <= SMALL_AREA), warp-cooperative (box <=
MEDIUM_MAX on both axes, not clipped), or the band queue and raster_band_kernel; each in 32-bit or 64-bit edge arithmetic by the
reach test; and back to the set-up kernel when the queues are full.  Every test asserts through path_census that its scene
reaches the paths it is about.  Depth, the shadow atlas and forward_stats()[:3] are integer artefacts: identical, not close."""
import numpy as np
import pytest

import raster_reference as ref
import raster_scenes as scenes
from rend3_b200 import glam
from rend3_b200.backend import load_cuda_backend
from rend3_b200.runner import TestRunner
from rend3_b200.world import BLEND, LEFT, Camera, MeshBuilder, Object, PbrMaterial

from oracle import load_oracle_backend

pytestmark = pytest.mark.gpu


@pytest.fixture()
def cuda():
    b = load_cuda_backend(0)
    yield b
    b.close()


def render_both(cuda, width, height, tris, z, samples, **kw):
    orc = load_oracle_backend()
    runners = []
    for b in (cuda, orc):
        r = scenes.build(b, width, height, tris, z, **kw)
        scenes.draw(r, width, height, samples)
        runners.append(r)
    return orc, runners[0]


def assert_parity(cuda, orc, what, runner=None):
    dc, do = cuda.readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32)
    assert np.array_equal(dc, do), f"{what}: {np.count_nonzero(dc != do)} depth texels differ from the oracle"
    sc, so = cuda.forward_stats(), orc.forward_stats()
    assert sc[:3] == so[:3], f"{what}: forward_stats {sc[:3]} against the oracle's {so[:3]}"
    if runner is not None and runner.last_eval.shadows:
        w, h = runner.last_eval.shadow_target_size
        ac, ao = cuda.readback_shadow_atlas(w, h).view(np.uint32), orc.readback_shadow_atlas(w, h).view(np.uint32)
        assert np.array_equal(ac, ao), f"{what}: {np.count_nonzero(ac != ao)} shadow atlas texels differ from the oracle"
        assert np.count_nonzero(ao) > 1000, f"{what}: the shadow pass drew nothing"
    return sc


@pytest.mark.parametrize("samples", [1, 4])
def test_path_boundaries(cuda, samples):
    """Boxes of exactly 64 and 65 pixels, 32x32 against 32x33 and 33x32, reach FITS32_REACH and one past it on the inline and the
    cooperative path, vertices on pixel centres and sample positions (top-left ties everywhere)."""
    tris, _ = scenes.boundary_scene()
    census = ref.path_census(scenes.snapped(tris), samples, (0, 0, 256, 256))
    assert all(census[k] > 0 for k in ("inline_int", "inline_ll", "coop_int", "coop_ll", "band")), census
    z = scenes.distinct_depths(len(tris), seed=2)
    orc, _ = render_both(cuda, 256, 256, tris, z, samples)
    assert_parity(cuda, orc, "boundary scene")
    assert scenes.assert_matches_reference(cuda, 256, 256, tris, z, samples, "boundary scene") > 0


@pytest.mark.parametrize("samples", [1, 4])
@pytest.mark.parametrize("cell,path", [(4, "inline_int"), (16, "coop_int"), (64, "band")])
def test_watertight_grid(cuda, cell, path, samples):
    """A jittered grid tiles the target: every sample covered exactly once, no depth texel left at the clear value."""
    tris = scenes.jittered_grid(256, cell, seed=cell)
    census = ref.path_census(scenes.snapped(tris), samples, (0, 0, 256, 256))
    assert census[path] > len(tris) // 2, census
    z = scenes.distinct_depths(len(tris), seed=cell)
    orc, _ = render_both(cuda, 256, 256, tris, z, samples)
    assert_parity(cuda, orc, f"grid {cell}")
    assert cuda.forward_stats()[1] == 256 * 256 * samples
    assert np.count_nonzero(cuda.readback_depth() == 0.0) == 0
    scenes.assert_matches_reference(cuda, 256, 256, tris, z, samples, f"grid {cell}")


@pytest.mark.parametrize("samples", [1, 4])
@pytest.mark.parametrize("cell", [4, 16, 64])
def test_watertight_blend_grid(cuda, cell, samples):
    """The blend routine over the same grids: one blended fragment per sample (forward_stats()[3]) and every pixel one translucent
    layer over the clear colour, evaluated by hand with rule R8."""
    import blend_case

    tris = scenes.jittered_grid(256, cell, seed=cell)
    r = scenes.build(cuda, 256, 256, tris, scenes.distinct_depths(len(tris), seed=cell), transparency=BLEND)
    scenes.draw(r, 256, 256, samples)
    assert cuda.forward_stats()[3] == 256 * 256 * samples
    want = np.array(blend_case.blend(scenes.COLOUR, [blend_case.f16(v) for v in scenes.CLEAR]), dtype=np.float32)
    hdr = cuda.readback_hdr_f32().reshape(-1, 4)
    assert np.array_equal(hdr, np.broadcast_to(want, hdr.shape)), f"{np.count_nonzero((hdr != want).any(axis=1))} pixels are not one layer"


# Along the shared diagonal the two triangles are clipped with clip_lerp from opposite ends, so in general the two clipped copies
# of the diagonal may round apart and leave gaps or double cover.  For this quad they do not: the oracle covers every sample exactly
# once at one and at four samples (measured), and the kernels must match it.
GUARD_QUAD_SLACK = 0


@pytest.mark.parametrize("samples", [1, 4])
def test_guard_band_clipping(cuda, samples):
    """Two triangles with vertices far beyond the 64x guard band, and long triangles whose clipped on-screen part has a medium
    pixel box: parity with the oracle, and the clipped quad covers the target once up to a stated slack along its diagonal."""
    subs = [s for t in scenes.GUARD_QUAD for s in ref.clip_to_guard_band(t, 256, 256)]
    census = ref.path_census(subs, samples, (0, 0, 256, 256), clipped=[True] * len(subs))
    assert census["band"] > 0, census
    orc, _ = render_both(cuda, 256, 256, scenes.GUARD_QUAD, [0.5, 0.5], samples)
    assert_parity(cuda, orc, "guard-band quad")
    assert abs(cuda.forward_stats()[1] - 256 * 256 * samples) <= GUARD_QUAD_SLACK * samples
    assert np.count_nonzero(cuda.readback_depth() == 0.0) == 0

    rng = np.random.default_rng(4)
    tris = []
    for _ in range(60):
        # two vertices within 24 pixels of an edge of the target, the third far beyond the guard band past that edge
        side = rng.integers(0, 4)
        u, v = float(rng.integers(8, 232)), float(rng.integers(4, 24))
        far = -1.0e5 if side < 2 else 1.0e5
        v = v if side < 2 else 256.0 - v
        tris.append(((v, u), (v, u + 16.0), (far, u + 8.0)) if side % 2 == 0 else ((u, v), (u + 16.0, v), (u + 8.0, far)))
    subs = [s for t in tris for s in ref.clip_to_guard_band(t, 256, 256)]
    census = ref.path_census(subs, samples, (0, 0, 256, 256), clipped=[True] * len(subs))
    unclipped = ref.path_census(subs, samples, (0, 0, 256, 256))
    assert census["band"] > 20 and unclipped["coop_int"] + unclipped["coop_ll"] > 20, (census, unclipped)
    orc, _ = render_both(cuda, 256, 256, tris, scenes.distinct_depths(len(tris), seed=4), samples)
    assert_parity(cuda, orc, "clipped medium sub-triangles")
    assert cuda.forward_stats()[1] > 0


@pytest.mark.parametrize("samples", [1, 4])
def test_near_plane_clipping(cuda, samples):
    """Perspective triangles crossing the near plane (R1's z >= 0 plane, new vertices interpolated in clip space)."""
    rng = np.random.default_rng(8)
    tris = []
    for _ in range(40):
        p = rng.uniform(-3.0, 3.0, (3, 3)).astype(np.float32)
        p[:, 2] = rng.uniform(-1.0, 6.0, 3)
        p[0, 2] = -abs(p[0, 2]) - 0.05   # one vertex behind the camera
        tris.append(p)
    orc = load_oracle_backend()
    for b in (cuda, orc):
        r = TestRunner(b, LEFT)
        mat = r.renderer.add_material(PbrMaterial(albedo_value=scenes.COLOUR, unlit=True))
        for p in tris:
            for order in ((0, 1, 2), (0, 2, 1)):   # both windings: whichever faces the camera is drawn
                m = MeshBuilder.new(p[list(order)], LEFT).with_vertex_normals(np.zeros((3, 3), np.float32)).build()
                r.renderer.add_object(Object(r.renderer.add_mesh(m), mat, glam.identity()))
        r.renderer.set_camera_data(Camera(("perspective", 60.0, 0.1), glam.identity()))
        r.render_frame(resolution=(256, 256), samples=samples)
    st = assert_parity(cuda, orc, "near plane")
    assert st[0] > 10 and st[1] > 1000


@pytest.mark.parametrize("samples", [1, 4])
def test_msaa_band_block_corners(cuda, samples):
    """Large triangles whose edges pass within a pixel of the 32 x 16 block corners: the band kernel's block skip (widened by
    k0..k2 for four samples) must never drop a covered sample."""
    tris = scenes.block_corner_triangles()
    census = ref.path_census(scenes.snapped(tris), samples, (0, 0, 256, 256))
    assert census["band"] == len(tris), census
    z = scenes.distinct_depths(len(tris), seed=6)
    orc, _ = render_both(cuda, 256, 256, tris, z, samples)
    assert_parity(cuda, orc, "block corners")
    scenes.assert_matches_reference(cuda, 256, 256, tris, z, samples, "block corners")


@pytest.mark.parametrize("samples", [1, 4])
def test_shadow_pass_and_cutout_on_every_path(cuda, samples):
    """The boundary scene in the shadow pass (depth mode) and with a textured cutout material (per-fragment alpha, MODE_ALPHA):
    atlas and depth identical to the oracle."""
    tris, _ = scenes.boundary_scene()
    z = scenes.distinct_depths(len(tris), seed=2)
    orc, r = render_both(cuda, 256, 256, tris, z, samples, cutout=True, shadow=True)
    assert_parity(cuda, orc, "cutout + shadow", runner=r)
    # the cutout really discards: fewer pixels than the opaque scene covers
    plain = load_oracle_backend()
    scenes.draw(scenes.build(plain, 256, 256, tris, z), 256, 256, samples)
    assert np.count_nonzero(orc.readback_depth()) < np.count_nonzero(plain.readback_depth()) - 500


@pytest.mark.parametrize("samples", [1, 4])
def test_degenerate_vertices_in_the_mesh(cuda, samples):
    """NaN, +-inf and 1e30 positions, vertices at w = 0 and behind the camera, and triangles whose vertices snap to one point:
    the kernels drop exactly what the oracle drops and rasterise the rest identically, without a fault."""
    rng = np.random.default_rng(12)
    good = rng.uniform(-2.0, 2.0, (64, 3, 3)).astype(np.float32)
    good[..., 2] = rng.uniform(1.0, 8.0, (64, 3))
    bad = good.copy()
    specials = [np.nan, np.inf, -np.inf, 1.0e30, -1.0e30]
    for i in range(64):
        k, axis = i % 3, (i // 3) % 3
        if i < 40:
            bad[i, k, axis] = specials[i % len(specials)]
        elif i < 48:
            bad[i, k, 2] = 0.0                                # w = 0 (view z = 0)
        elif i < 56:
            bad[i, k, 2] = -rng.uniform(0.5, 3.0)             # behind the camera
        else:
            bad[i, 1] = bad[i, 0] + np.float32(1e-6)          # the three vertices snap to one point
            bad[i, 2] = bad[i, 0] - np.float32(1e-6)
    orc = load_oracle_backend()
    for b in (cuda, orc):
        r = TestRunner(b, LEFT)
        mat = r.renderer.add_material(PbrMaterial(albedo_value=scenes.COLOUR, unlit=True))
        pos = np.concatenate([good, bad, bad[:, [0, 2, 1]]]).reshape(-1, 3)
        m = MeshBuilder.new(pos, LEFT).with_vertex_normals(np.zeros_like(pos)).build()
        h = r.renderer.add_object(Object(r.renderer.add_mesh(m), mat, glam.identity()))
        rec = r.renderer.objects[h]["rec"]   # the mesh's bounding sphere is NaN: give the object one that is always visible
        rec["sphere_center"], rec["sphere_radius"] = (0.0, 0.0, 0.0), 1.0e4
        r.renderer.set_camera_data(Camera(("perspective", 60.0, 0.1), glam.identity()))
        r.render_frame(resolution=(256, 256), samples=samples)
    st = assert_parity(cuda, orc, "degenerate vertices")
    assert st[0] > 10 and st[1] > 0


# ------------------------------------------------------------------ queue-full fallbacks
def slivers(n, width, x_step, rows_from, rows_to):
    """n right triangles one pixel wide from row `rows_from` to `rows_to` (pixels), in columns 0, x_step, 2 x_step, ..."""
    x = (np.arange(n) * x_step) % width
    t = np.zeros((n, 3, 2))
    t[:, 0] = np.stack([x, np.full(n, rows_from)], 1)
    t[:, 1] = np.stack([x + 1.0, np.full(n, rows_from)], 1)
    t[:, 2] = np.stack([x, np.full(n, rows_to)], 1)
    return scenes.oriented(t)


@pytest.mark.parametrize("samples", [1, 4])
def test_band_queue_overflow(cuda, samples):
    """More than BAND_CAP band items in one pass.  90,000 full-height slivers of 192 band items (frame 1) and, moved down 8 rows
    and right half a pixel, of 193 (frame 2): neither count divides BAND_CAP, so in each frame one reservation straddles the cap
    and leaves slots below it that the band kernel would read.  Frame 2's straddling slots held frame 1's items.  Depth identical
    to the oracle, and the covered-sample count equal to the oracle's and to the exact reference (a stale item would add samples)."""
    n, width, height = 90_000, 256, 4096
    tris = slivers(n, width, 1, 0.0, 3071.5)
    moved = tris + np.array([0.5, 8.0])
    rect = (0, 0, width, height)
    for t, nb in ((tris, 192), (moved, 193)):
        census = ref.path_census(scenes.snapped(t[:1]), samples, rect)
        assert census["band"] == 1 and census["band_items"] == nb
        assert n * nb > ref.BAND_CAP and ref.BAND_CAP % nb != 0
    z = np.random.default_rng(3).integers(1, 1 << 12, n).astype(np.float32) / np.float32(1 << 12)
    orc = load_oracle_backend()
    runners = [scenes.build(b, width, height, tris, z) for b in (cuda, orc)]
    for frame, t in enumerate((tris, moved)):
        for b, r in zip((cuda, orc), runners):
            if frame:
                r.renderer.set_object_transform(r.object, glam.from_translation((0.5, 8.0, 0.0)))
            scenes.draw(r, width, height, samples)
        st = assert_parity(cuda, orc, f"band overflow frame {frame}")
        assert st[1] == ref.covered_count(scenes.snapped(t), width, height, samples), f"frame {frame}"


@pytest.mark.parametrize("samples", [1, 4])
def test_large_queue_overflow(cuda, samples):
    """More than LARGE_CAP large sub-triangles in one pass: 4.3 M slivers of 33 x 3 pixels, each one band item on the band path.
    The ones past the cap are handed to the warp; nothing is lost or drawn twice."""
    n, size = 4_300_000, 256
    rng = np.random.default_rng(7)
    x = rng.integers(0, size - 34, n).astype(np.float64)
    y = (rng.integers(0, size // 16, n) * 16 + rng.integers(0, 13, n)).astype(np.float64)
    t = np.zeros((n, 3, 2))
    t[:, 0] = np.stack([x, y], 1)
    t[:, 1] = np.stack([x + 33.0, y], 1)
    t[:, 2] = np.stack([x, y + 3.0], 1)
    t = scenes.oriented(t)
    census = ref.path_census(scenes.snapped(t[:64]), samples, (0, 0, size, size))
    assert census["band"] == 64 and census["band_items"] == 64 and n > ref.LARGE_CAP
    z = rng.integers(1, 1 << 12, n).astype(np.float32) / np.float32(1 << 12)
    orc, _ = render_both(cuda, size, size, t, z, samples)
    st = assert_parity(cuda, orc, "large overflow")
    assert st[1] == ref.covered_count(scenes.snapped(t), size, size, samples)
