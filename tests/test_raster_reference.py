"""The CPU oracle's rasteriser against the exact coverage reference (tests/raster_reference.py) on scenes with exactly snapped
vertices, and the reference itself against hand-computed answers.  No GPU needed: this pins the oracle on its own terms, not
only through the reference's golden images."""
import numpy as np
import pytest

import raster_reference as ref
import raster_scenes as scenes
from rend3_b200.world import BLEND

from oracle import load_oracle_backend


def px(x, y):
    """Sub-pixel integers of a point given in pixels."""
    return (int(round(x * 256)), int(round(y * 256)))


def covered_pixels(tri, size, samples=1):
    _, owner = ref.coverage([tri], size, size, samples)
    return {(int(x), int(y)) for y, x in zip(*np.nonzero((owner >= 0).any(axis=2)))}, owner


def test_reference_top_left_known_answers():
    """Hand-evaluated ties.  The square with corners on the pixel centres (0.5, 0.5) and (2.5, 2.5), split along its diagonal:
    the centres on its top and left sides belong to it, those on its bottom and right sides do not, and each centre on the shared
    diagonal belongs to exactly one half."""
    upper = (px(0.5, 0.5), px(2.5, 0.5), px(0.5, 2.5))     # top and left sides, the diagonal is its bottom-right edge
    lower = (px(2.5, 0.5), px(2.5, 2.5), px(0.5, 2.5))     # right and bottom sides, the diagonal is its top-left edge
    assert covered_pixels(upper, 4)[0] == {(0, 0), (1, 0), (0, 1)}
    assert covered_pixels(lower, 4)[0] == {(1, 1)}
    # the opposite winding covers the same samples (the kernels orient before testing)
    assert covered_pixels(upper[::-1], 4)[0] == {(0, 0), (1, 0), (0, 1)}
    # a horizontal edge through sample 0 of row 0 (y = 32 sub-pixels): on a top edge the sample is in, on a bottom edge it is out
    top = ((0, 32), (4 * 256, 32), (0, 4 * 256))
    bottom = ((0, 32), (4 * 256, -4 * 256), (4 * 256, 32))
    _, o_top = covered_pixels(top, 4, samples=4)
    _, o_bottom = covered_pixels(bottom, 4, samples=4)
    assert o_top[0, 0].tolist() == [0, 0, 0, 0] and o_top[0, 2].tolist() == [0, 0, 0, 0]
    assert o_bottom[0, 1].tolist() == [-1, -1, -1, -1]      # samples 1..3 lie below y = 32, sample 0 on the bottom edge
    # a vertical edge x = 32 through sample 2 of column 0, whose other samples lie to its right: on a left edge (interior to
    # the right) all four samples are in, on a right edge (interior to the left) none is
    left = ((32, 0), (32 + 4 * 256, 4 * 256), (32, 4 * 256))
    _, o_left = ref.coverage([left], 4, 4, 4)
    assert o_left[3, 0].tolist() == [0, 0, 0, 0]
    right = ((32, 0), (32, 4 * 256), (32 - 4 * 256, 4 * 256))
    _, o_right = ref.coverage([right], 4, 4, 4)
    assert o_right[3, 0].tolist() == [-1, -1, -1, -1]
    # the same right edge one pixel further (x = 288): column 1 has sample 2 on it and the others beyond it, column 0 is inside
    _, o_right = ref.coverage([tuple((x + 256, y) for x, y in right)], 4, 4, 4)
    assert o_right[3, 1].tolist() == [-1, -1, -1, -1] and o_right[3, 0].tolist() == [0, 0, 0, 0]
    # zero area covers nothing; a pixel-sized square of two triangles covers its one centre once
    assert ref.coverage([(px(0, 0), px(1, 1), px(2, 2))], 4, 4, 1)[0] == 0
    quad = [(px(1, 1), px(2, 1), px(2, 2)), (px(1, 1), px(2, 2), px(1, 2))]
    assert ref.coverage(quad, 4, 4, 1)[0] == 1 and ref.coverage(quad, 4, 4, 4)[0] == 4


def test_reference_helpers_agree():
    """covered_count's shape sharing equals the per-triangle count; plane_depth interpolates a tilted plane exactly."""
    tris = scenes.snapped(scenes.jittered_grid(64, 16, seed=3))
    shifted = np.concatenate([tris + 256 * 7, tris[:5] + [256 * 3, 256 * 2]])
    for samples in (1, 4):
        assert ref.covered_count(shifted, 128, 128, samples) == ref.coverage(shifted, 128, 128, samples)[0]
    tri = (px(0, 0), px(8, 0), px(0, 8))
    d = ref.plane_depth(tri, (0.5, 0.75, 0.25), np.array([4 * 256.0, 0.0]), np.array([0.0, 4 * 256.0]))
    assert np.allclose(d, [0.625, 0.375], rtol=0, atol=1e-15)


@pytest.mark.parametrize("samples", [1, 4])
def test_census_reaches_every_path(samples):
    """The boundary scene puts triangles on both sides of each threshold of r3_raster.cu's path choice."""
    tris, labels = scenes.boundary_scene()
    census = ref.path_census(scenes.snapped(tris), samples, (0, 0, 256, 256))
    per = dict(zip(labels, census["per_triangle"]))
    for key in ("inline_int", "inline_ll", "coop_int", "coop_ll", "band"):
        assert census[key] > 0, (key, census)
    for k in range(4):
        assert per[f"box 8x8 corner {k}"] == per[f"box 16x4 corner {k}"] == per[f"box 32x2 corner {k}"] == "inline_int"     # 64 px
        assert per[f"box 13x5 corner {k}"] == per[f"box 5x13 corner {k}"] == per[f"box 32x32 corner {k}"] == "coop_int"    # 65 px .. 32x32
        assert per[f"box 33x2 corner {k}"] == per[f"box 32x33 corner {k}"] == per[f"box 33x32 corner {k}"] == "band"
    for axis in ("x", "y"):
        assert per[f"inline reach {ref.FITS32_REACH} along {axis}"] == "inline_int"
        assert per[f"inline reach {ref.FITS32_REACH + 1} along {axis}"] == "inline_ll"
        assert per[f"coop reach {ref.FITS32_REACH} along {axis}"] == "coop_int"
        assert per[f"coop reach {ref.FITS32_REACH + 1} along {axis}"] == "coop_ll"
    assert not census["queue_full"]


def test_census_of_clipped_medium_triangles():
    """A triangle reaching beyond the guard band is clipped; its on-screen sub-triangles have a medium pixel box but take the band
    queue, because the set-up kernel hands only unclipped triangles to the warp."""
    tri = [(8.0, 8.0), (8.0, 24.0), (-100000.0, 16.0)]
    subs = ref.clip_to_guard_band(tri, 256, 256)
    assert len(subs) == 2
    census = ref.path_census(subs, 1, (0, 0, 256, 256), clipped=[True] * len(subs))
    unclipped = ref.path_census(subs, 1, (0, 0, 256, 256))
    assert census["band"] == 2 and unclipped["coop_int"] + unclipped["coop_ll"] == 2


@pytest.mark.parametrize("samples", [1, 4])
def test_oracle_boundary_scene_matches_reference(samples):
    tris, _ = scenes.boundary_scene()
    z = scenes.distinct_depths(len(tris), seed=2)
    b = load_oracle_backend()
    scenes.draw(scenes.build(b, 256, 256, tris, z), 256, 256, samples)
    scenes.assert_matches_reference(b, 256, 256, tris, z, samples, "oracle boundary scene")


@pytest.mark.parametrize("samples", [1, 4])
@pytest.mark.parametrize("cell", [4, 16, 64])
def test_oracle_jittered_grid_matches_reference(cell, samples):
    """The grid tiles the target: every sample is covered exactly once."""
    tris = scenes.jittered_grid(128, cell, seed=cell)
    z = scenes.distinct_depths(len(tris), seed=cell)
    b = load_oracle_backend()
    scenes.draw(scenes.build(b, 128, 128, tris, z), 128, 128, samples)
    assert scenes.assert_matches_reference(b, 128, 128, tris, z, samples, f"oracle grid {cell}") == 128 * 128 * samples


@pytest.mark.parametrize("samples", [1, 4])
def test_oracle_block_corner_triangles_match_reference(samples):
    tris = scenes.block_corner_triangles()
    z = scenes.distinct_depths(len(tris), seed=6)
    b = load_oracle_backend()
    scenes.draw(scenes.build(b, 256, 256, tris, z), 256, 256, samples)
    scenes.assert_matches_reference(b, 256, 256, tris, z, samples, "oracle block corners")


def test_oracle_blend_grid_known_answer():
    """The blend routine over a tiling grid: one blended fragment per sample, each pixel one layer over the clear colour (rule R8)."""
    import blend_case

    tris = scenes.jittered_grid(64, 16, seed=9)
    b = load_oracle_backend()
    scenes.draw(scenes.build(b, 64, 64, tris, scenes.distinct_depths(len(tris)), transparency=BLEND), 64, 64, 1)
    assert b.forward_stats()[3] == 64 * 64
    want = np.array(blend_case.blend(scenes.COLOUR, [blend_case.f16(v) for v in scenes.CLEAR]), dtype=np.float32)
    assert np.array_equal(b.readback_hdr_f32().reshape(-1, 4), np.broadcast_to(want, (64 * 64, 4)))
