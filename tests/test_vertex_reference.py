"""The vertex stage (vs_main's attribute half, R6 interpolation, the normal-map tangent basis) against the float64 restatement of
tests/vertex_reference.py, on the scenes of tests/vertex_scenes.py: the CPU oracle without a GPU, and on the GPU the kernels of
rend3_b200/csrc/r3_shade.cu (resolve_kernel<1|4, TEX> and blend_apply_kernel).

The bound is TOL (relative above 1.0) plus the sensitivity allowance of tests/shade_reference.py, widened by the f32 rounding of
the R6 weights carried through fs_main, plus the rgba16f rounding of each sample at 4x.  NaN equals NaN.  A census per scene
asserts that the case it exists for is reached: pixels where inv_scale_sq := 1 would move the value beyond the bound, pixels on
clipped triangles, 4x pixels whose primitive is shaded at a centre it does not cover, every normal-map layout, and NaN normals."""
import functools

import numpy as np
import pytest

import shade_reference as ref
import vertex_reference as vref
import vertex_scenes as vs
from rend3_b200.layouts import MAT_BICOMPONENT_NORMAL, MAT_SWIZZLED_NORMAL, MAT_YDOWN_NORMAL

from oracle import load_oracle_backend

# unlit vertex colours depend on the weights and the colour bytes alone: 1e-6 plus the f32 rounding allowance of the R6 weights
# (the oracle's largest error is 7e-5, on triangles seen edge-on, where the cross products cancel; every error is inside the allowance)
UNLIT_BOUND = 1e-6


def atlas(backend, runner):
    w, h = runner.last_eval.shadow_target_size
    return backend.readback_shadow_atlas(w, h)


@functools.lru_cache(maxsize=None)
def oracle_case(name, samples):
    """(scene, oracle backend, expected) of a scene rendered by the oracle."""
    scene = vs.SCENES[name]()
    o = load_oracle_backend()
    r = vs.render(o, scene, samples, texture_table=vs.needs_texture_table(scene))
    return scene, o, vs.expected(scene, o, r, samples, atlas(o, r))


# ------------------------------------------------------------------ the reference itself
def test_reference_known_answers():
    # a sheared mv3: columns (2, 0, 0), (1, 1, 0), (0, 0, 1).  inv_scale_sq = (1/4, 1/2, 1) per COLUMN; the normal (0, 1, 0)
    # becomes mv3 * (0, 1/2, 0) = (1/2, 1/2, 0), normalised (1, 1, 0) / sqrt(2) - not the inverse transpose's (-1, 2, 0) / sqrt(5)
    mv = np.eye(4, dtype=np.float32)
    mv[0, 0], mv[1, 0] = 2.0, 1.0
    assert vref.inv_scale_squared(mv.reshape(16)).tolist() == [0.25, 0.5, 1.0]
    n = vref.transform_direction(mv.reshape(16), np.array([[0.0, 1.0, 0.0]]))
    assert np.allclose(n, [[2 ** -0.5, 2 ** -0.5, 0.0]], rtol=0, atol=1e-15)
    # a zero column: 1 / 0 = inf, inf * 0 = NaN
    z = np.eye(4, dtype=np.float32)
    z[2, 2] = 0.0
    assert np.isinf(vref.inv_scale_squared(z.reshape(16))[2]) and np.isnan(vref.transform_direction(z.reshape(16), np.array([[0.0, 1.0, 0.0]]))).all()
    # R6: the vertices (0, 0, 1), (1, 0, 1), (0, 2, 2) in clip xyw, i.e. ndc (0, 0), (1, 0), (0, 1); at ndc (0.25, 0.25) the
    # screen-space weights (1/2, 1/4, 1/4) are divided by w and renormalised: (1/2, 1/4, 1/8) / (7/8)
    p = np.array([[0.0, 0.0, 1.0], [1.0, 0.0, 1.0], [0.0, 2.0, 2.0]])
    assert np.allclose(vref.weights(p, np.array([0.25]), np.array([0.25])), [[4 / 7, 2 / 7, 1 / 7]], rtol=0, atol=1e-15)
    # outside the triangle a weight is negative: extrapolation
    assert vref.weights(p, np.array([1.0]), np.array([0.5]))[0, 0] < 0.0
    # the ndc of a pixel centre
    assert vref.ndc(np.array([0.5]), np.array([0.5]), 4, 2) == (np.array([-0.75]), np.array([0.5]))
    # the TBN of an orthonormal frame t = x, n = z: b = cross(n, t) = y, so the map value comes out unchanged
    m = np.array([[0.6, 0.0, 0.8]])
    assert np.allclose(vref.tbn_normal(np.array([[0.0, 0.0, 3.0]]), np.array([[2.0, 0.0, 0.0]]), m), m, rtol=0, atol=1e-15)
    # and turned by 90 degrees about z (t = y, n = z, b = -x)
    assert np.allclose(vref.tbn_normal(np.array([[0.0, 0.0, 1.0]]), np.array([[0.0, 1.0, 0.0]]), m), [[0.0, 0.6, 0.8]], rtol=0, atol=1e-15)
    # the map value per layout (texel 0.5 -> 0, 1 -> 1), y-down negates y, the swizzle takes x from alpha
    t = np.array([[1.0, 0.5, 0.5, 0.5]])
    assert np.allclose(vref.normal_map_value(t, 0), [[1.0, 0.0, 0.0]])
    assert np.allclose(vref.normal_map_value(np.array([[0.5, 0.75, 0.0, 1.0]]), MAT_BICOMPONENT_NORMAL | MAT_YDOWN_NORMAL), [[0.0, -0.5, 0.75 ** 0.5]])
    assert np.allclose(vref.normal_map_value(np.array([[0.5, 0.5, 0.0, 1.0]]), MAT_BICOMPONENT_NORMAL | MAT_SWIZZLED_NORMAL), [[1.0, 0.0, 0.0]])
    # colour bytes: byte 0 is red; absent colour is 1, absent tangent 0
    assert np.allclose(vref.unpack_colour(np.array([[10, 20, 30, 40]], dtype=np.uint8), 1), [[10 / 255, 20 / 255, 30 / 255, 40 / 255]])
    assert vref.unpack_colour(None, 2).tolist() == [[1.0] * 4] * 2 and vref.attribute(None, 1, 3).tolist() == [[0.0] * 3]


# ------------------------------------------------------------------ the oracle
@pytest.mark.parametrize("samples", [1, 4])
@pytest.mark.parametrize("name", list(vs.SCENES))
def test_oracle_matches_vertex_reference(name, samples):
    """Every decided pixel within the bound; decided pixels are covered (or not) as the depth readback says, uncovered ones keep
    the clear colour; fewer than 5 % of the values need more than TOL."""
    scene, o, e = oracle_case(name, samples)
    hdr, depth = o.readback_hdr_f32(), o.readback_depth()
    bad, n, needed = vs.compare(hdr, e)
    assert n > 0 and not bad.any(), f"{name} {samples}x: {bad.any(axis=2).sum()} pixels outside the bound, first at {np.argwhere(bad)[0]}"
    assert np.all(depth[e.keep & e.covered] > 0) and np.all(depth[e.keep & e.empty] == 0), "coverage differs from the depth readback"
    clear = np.float32(vs.CLEAR) if samples == 1 else np.float16(vs.CLEAR).astype(np.float32)
    assert np.all(hdr[e.keep & e.empty] == clear)
    assert needed < 0.05, f"{needed:.2%} of the values needed the allowance"
    assert np.count_nonzero(e.keep & ~e.empty) > 1000


def test_unlit_vertex_colours_tight():
    """Unlit vertex-coloured materials return the interpolated colour times the albedo: a check of the weights and the byte order
    alone, to UNLIT_BOUND (absolute) instead of TOL."""
    for name in ("spheres_lh", "spheres_rh"):
        scene, o, e = oracle_case(name, 1)
        m = e.keep & e.unlit
        assert np.count_nonzero(m) > 200
        excess = np.abs(o.readback_hdr_f32()[m] - e.want[m]) - e.sens[m]
        assert excess.max() <= UNLIT_BOUND, f"{name}: {excess.max():.3e}"


CENSUS = {
    "spheres_lh": dict(iss=200, clipped=1000, unlit=200),
    "spheres_rh": dict(iss=200, clipped=1000, unlit=200),
    "normal_maps_lh": dict(iss=200, layouts=50),
    "normal_maps_rh": dict(iss=200, layouts=50),
    "ieee": dict(nan=("zero_normal", "zero_scale", "nmap_no_uv")),
}


@pytest.mark.parametrize("name", list(vs.SCENES))
def test_scene_census(name):
    """Each scene reaches the case it exists for, on pixels that are compared."""
    want = CENSUS[name]
    for samples in (1, 4):
        _, _, e = oracle_case(name, samples)
        k = e.keep
        if "iss" in want:
            assert np.count_nonzero(k & e.iss_moves) >= want["iss"], "inv_scale_sq := 1 changes too few pixels"
        if "clipped" in want:
            assert np.count_nonzero(k & e.clipped) >= want["clipped"], "too few pixels on clipped triangles"
        if "unlit" in want:
            assert np.count_nonzero(k & e.unlit) >= want["unlit"]
        if "layouts" in want:
            for layout in vs.NORMAL_LAYOUTS:
                assert np.count_nonzero(k & (e.label == f"nmap_{layout}")) >= want["layouts"], layout
            assert np.count_nonzero(k & np.char.endswith(e.label.astype(str), "_generated")) >= want["layouts"]
        if "nan" in want:
            for label in want["nan"]:
                assert np.count_nonzero(k & e.nan & (e.label == label)) >= 100, label
        if samples == 4:
            assert np.count_nonzero(k & e.extrapolated) >= 100, "too few 4x pixels shaded at an uncovered centre"


# ------------------------------------------------------------------ the kernels
@pytest.fixture()
def cuda():
    from rend3_b200.backend import load_cuda_backend
    b = load_cuda_backend(0, parity_target=True)
    yield b
    b.close()


def assert_close_to_oracle(a, o, e, what, steps=0):
    """The kernel within TOL + allowance (+ f16, + `steps` half-precision steps) of the oracle wherever one object covers the pixel
    (NaN equals NaN)."""
    bound = ref.TOL * np.maximum(1.0, np.abs(o)) + np.nan_to_num(e.sens) + e.f16 * 2 + steps * vs.f16_step(o)
    bad = ~(np.abs(a - o) <= bound) & ~(np.isnan(a) & np.isnan(o)) & e.single[..., None]
    assert not bad.any(), f"{what}: {bad.any(axis=2).sum()} pixels differ from the oracle, first at {np.argwhere(bad)[0]}"


GPU_CASES = [(n, s, t) for n in vs.SCENES for s in (1, 4) for t in ((True,) if vs.needs_texture_table(vs.SCENES[n]()) else (False, True))]


@pytest.mark.gpu
@pytest.mark.parametrize("name,samples,tex", GPU_CASES)
def test_kernel_matches_vertex_reference(cuda, name, samples, tex):
    """resolve_kernel<samples, tex>: depth and the shadow atlas bit-identical to the oracle, pixels within the bound of the reference
    and of the oracle."""
    scene = vs.SCENES[name]()
    rc = vs.render(cuda, scene, samples, texture_table=tex)
    o = load_oracle_backend()
    ro = vs.render(o, scene, samples, texture_table=tex)
    ac, ao = atlas(cuda, rc), atlas(o, ro)
    assert np.array_equal(ac.view(np.uint32), ao.view(np.uint32)), "shadow atlas differs from the oracle"
    dc, do = cuda.readback_depth(), o.readback_depth()
    assert np.array_equal(dc.view(np.uint32), do.view(np.uint32)), f"{np.count_nonzero(dc != do)} depth texels differ from the oracle"
    e = vs.expected(scene, cuda, rc, samples, ac, with_census=False)
    a = cuda.readback_hdr_f32().astype(np.float64)
    bad, n, needed = vs.compare(a, e)
    print(f"{name} {samples}x tex={tex}: {n} values, {needed:.3%} needed more than TOL")
    assert n > 0 and not bad.any(), f"{bad.any(axis=2).sum()} pixels outside the reference's bound, first at {np.argwhere(bad)[0]}"
    assert needed < 0.05
    assert_close_to_oracle(a, o.readback_hdr_f32().astype(np.float64), e, f"{name} {samples}x tex={tex}")
    if samples == 1 and name.startswith("spheres"):
        m = e.keep & e.unlit
        assert (np.abs(a[m] - e.want[m]) - e.sens[m]).max() <= UNLIT_BOUND


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["spheres_lh", "spheres_rh"])
def test_blend_matches_vertex_reference(cuda, name):
    """blend_apply_kernel: a translucent copy (alpha 0.4, scaled 1.08 about its centre) of every sphere, at 1x.  Where one copy lies
    over its own sphere or over the clear colour, the target holds src * a + f16(dst) * (1 - a) by rule R8."""
    scene = vs.SCENES[name]()
    rc = vs.render(cuda, scene, 1, translucent=0.4)
    o = load_oracle_backend()
    vs.render(o, scene, 1, translucent=0.4)
    assert np.array_equal(cuda.readback_depth().view(np.uint32), o.readback_depth().view(np.uint32))
    assert cuda.forward_stats()[3] > 0
    ac = atlas(cuda, rc)
    objs = vs.all_objects(scene, 0.4)
    back = vs.expected(scene, cuda, rc, 1, ac, objs=scene.objects, with_census=False)
    front = vs.expected(scene, cuda, rc, 1, ac, objs=objs, with_census=False)     # the nearest layer: the translucent copy
    over = np.char.endswith(front.label.astype(str), "_blend") & ((back.label == "") | (np.char.add(back.label.astype(str), "_blend") == front.label.astype(str)))
    src, a = front.want, front.want[..., 3:]
    dst = np.float16(back.want).astype(np.float64)
    want = np.concatenate([src[..., :3] * a + dst[..., :3] * (1.0 - a), a + dst[..., 3:] * (1.0 - a)], axis=-1)
    sens = a * front.sens + (1.0 - a) * back.sens
    got = cuda.readback_hdr_f32().astype(np.float64)
    one_layer = vs.layers(scene, cuda, objs, range(len(scene.objects), len(objs))) == 1     # translucent copies may overlap
    keep = front.keep & back.keep & over & one_layer
    bound = ref.TOL * np.maximum(1.0, np.abs(want)) + 2.0 * vs.f16_step(want) + sens
    bad = ~(np.abs(got - want) <= bound) & keep[..., None]
    assert np.count_nonzero(keep) > 300 and not bad.any(), f"{bad.any(axis=2).sum()} blended pixels outside the bound"
    assert_close_to_oracle(got, o.readback_hdr_f32().astype(np.float64), front, f"{name} blend", steps=2)
