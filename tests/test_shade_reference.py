"""The CPU oracle's fs_main against the float64 shading reference (tests/shade_reference.py) on the scenes of
tests/shade_scenes.py, and the reference itself against hand-evaluated answers.  No GPU needed: this pins the oracle's shading on
its own terms, beyond the reference's three lit golden images, before any kernel is compared with it."""
import numpy as np
import pytest

import shade_reference as ref
import shade_scenes as scenes
from rend3_b200.world import PbrMaterial

from oracle import load_oracle_backend


def records(*materials):
    return np.stack([m.to_record() for m in materials])


def one(mat, vp, normal, **kw):
    return ref.fs_main(np.array([vp], dtype=np.float64), np.array([normal], dtype=np.float64), records(mat), np.ones((1, 4)),
                       kw.pop("ambient", (0.0, 0.0, 0.0, 0.0)), **kw)[0]


def test_lambert_known_answer():
    """Reflectance 0 and metallic 0 make f0 = f90 = 0: only Lambert is left, albedo / pi * I * n.l."""
    albedo = (0.5, 0.25, 1.0, 1.0)
    m = PbrMaterial(albedo_value=albedo, roughness_factor=0.5, reflectance=0.0)
    l = np.array([0.0, 0.6, -0.8])
    got = one(m, (3.0, 4.0, 12.0), (0.0, 0.0, -1.0), dir_l=[l], dir_color=[(2.0, 1.0, 0.5)])
    nol = 0.8   # l is rounded to f32 like the light record: 1e-7 relative
    want = np.float32(albedo[:3]).astype(np.float64) / ref.PI * np.array([2.0, 1.0, 0.5]) * nol
    assert np.allclose(got[:3], want, rtol=1e-7, atol=0) and got[3] == np.float32(albedo[3])
    # the same with a point light at distance 1 of radius 2: att = (1 - 1/4)^2 / (1 + 1/4) = 0.45
    vp = np.array([3.0, 4.0, 12.0])
    got = one(m, vp, (0.0, 0.0, -1.0), pl_pos=[vp + 1.0 * l], pl_color=[(2.0, 1.0, 0.5)], pl_radius=[2.0])
    assert np.allclose(got[:3], want * 0.45, rtol=1e-7, atol=0)


def test_light_at_its_radius_contributes_nothing():
    m = PbrMaterial(albedo_value=(0.8, 0.8, 0.8, 1.0), roughness_factor=0.3)
    vp = np.array([10.5, 20.5, 5.0])
    lit = one(m, vp, (0.0, 0.0, -1.0), pl_pos=[vp + (0.0, 3.0, -4.0)], pl_color=[(1.0, 1.0, 1.0)], pl_radius=[5.001])
    assert lit[:3].min() > 0.0
    at = one(m, vp, (0.0, 0.0, -1.0), pl_pos=[vp + (0.0, 3.0, -4.0)], pl_color=[(1.0, 1.0, 1.0)], pl_radius=[5.0])
    assert at[:3].tolist() == [0.0, 0.0, 0.0]
    assert ref.point_attenuation(np.array([5.0, 7.0, 0.0]), 5.0).tolist() == [0.0, 0.0, 1.0]
    # a negative or NaN radius saturates d / radius to 0 (minNum / maxNum): attenuation 1 at any distance
    assert ref.point_attenuation(np.array([1e6]), -3.0)[0] == 1.0 and ref.point_attenuation(np.array([1e6]), np.nan)[0] == 1.0


def test_unlit_returns_albedo_and_ambient_floor():
    m = PbrMaterial(albedo_value=(0.2, 0.4, 0.6, 0.5), unlit=True)
    got = one(m, (1.0, 1.0, 1.0), (0.0, 0.0, -1.0), dir_l=[(0.0, 0.0, -1.0)], dir_color=[(5.0, 5.0, 5.0)], ambient=(1, 1, 1, 1))
    assert got.tolist() == np.float32([0.2, 0.4, 0.6, 0.5]).astype(np.float64).tolist()
    # lit, facing away from its only light: the colour is max(ambient * albedo, 0)
    lit = PbrMaterial(albedo_value=(0.2, 0.4, 0.6, 0.5), roughness_factor=0.5)
    got = one(lit, (1.0, 1.0, 1.0), (0.0, 0.0, -1.0), dir_l=[(0.0, 0.0, 1.0)], dir_color=[(5.0, 5.0, 5.0)], ambient=(0.5, 0.25, 0.1, 0.0))
    want = np.float32([0.2, 0.4, 0.6]).astype(np.float64) * np.float32([0.5, 0.25, 0.1]).astype(np.float64)
    assert np.allclose(got[:3], want, rtol=1e-15) and got[3] == np.float32(0.5)


def test_clear_coat_remap():
    """perceptual * (1 - cc) + max(perceptual, cc_rough) * cc, and nothing when cc == 0."""
    assert ref.clear_coat_remap(np.array([0.2]), np.array([0.5]), np.array([0.8]))[0] == pytest.approx(0.5)
    assert ref.clear_coat_remap(np.array([0.6]), np.array([0.5]), np.array([0.1]))[0] == pytest.approx(0.6)
    assert ref.clear_coat_remap(np.array([0.6]), np.array([0.0]), np.array([0.9]))[0] == 0.6
    assert ref.clear_coat_remap(np.array([0.5]), np.array([-1.0]), np.array([1.0]))[0] == 0.0
    px = ref.Pixel(records(PbrMaterial(roughness_factor=0.2, clearcoat_factor=0.5, clearcoat_roughness_factor=0.8)), np.ones((1, 4)),
                   np.array([[0.0, 0.0, -1.0]]))
    assert px.roughness[0] == pytest.approx((0.2 * 0.5 + 0.8 * 0.5) ** 2, rel=1e-6)


def test_pcf5_known_answers():
    atlas = np.zeros((8, 8))
    atlas[:, 4:] = 0.5
    # the centre of texel (2, 3): every tap sits on a texel centre, all ten texels are 0 -> lit
    f, margin = ref.pcf5(atlas, np.array([2.5 / 8]), np.array([3.5 / 8]), np.array([0.25]))
    assert f[0] == 1.0 and margin[0] == 0.25
    # the centre of texel (3, 3): the +x tap reads column 4, which holds 0.5 > ref -> one tap in five is shadowed
    f, _ = ref.pcf5(atlas, np.array([3.5 / 8]), np.array([3.5 / 8]), np.array([0.25]))
    assert f[0] == pytest.approx(0.8)
    # half-way between texel centres 3 and 4: the centre tap is half lit, the +x tap shadowed, the -x tap lit, +-y half lit
    f, _ = ref.pcf5(atlas, np.array([4.0 / 8]), np.array([3.5 / 8]), np.array([0.25]))
    assert f[0] == pytest.approx((0.5 + 0.5 + 0.5 + 0.0 + 1.0) / 5)


SCENES = {
    "grid_40_point_3_dir": lambda: scenes.grid_with_lights(40, 3),
    "grid_roughness_1e-10": lambda: scenes.grid_with_lights(20, 2, seed=3, roughness=1e-10),
    "half_covered_tiles": scenes.half_covered_layout,
    "pythagorean": scenes.pythagorean_layout,
    "far_small_radii": scenes.far_layout,
    **{f"tangent_{f!r}": (lambda f=f: scenes.tangent_layout(f)) for f in scenes.TANGENT_FACTORS},
    **{f"degenerate_{k}": (lambda k=k: scenes.degenerate_light_scene(k)) for k in scenes.DEGENERATE_KINDS},
    **{f"shadow_{n}_dir": (lambda n=n: scenes.shadow_scene(n)) for n in (1, 8, 9, 12)},
}


def oracle_frame(scene, samples, **kw):
    o = load_oracle_backend()
    o.runner = scenes.render(o, scene, samples, **kw)
    return o


@pytest.mark.parametrize("samples", [1, 4])
@pytest.mark.parametrize("name", list(SCENES))
def test_oracle_matches_shading_reference(name, samples):
    """Every covered pixel within TOL plus the sensitivity allowance of the float64 fs_main, except where a shadow lookup is
    decided by 1e-5 or less; uncovered pixels keep the clear colour.  On the material grid fewer than 5 % of the values may need
    the allowance, so the bound is not vacuous."""
    scene = SCENES[name]()
    o = oracle_frame(scene, samples)
    w, h = o.runner.last_eval.shadow_target_size
    e = scenes.expected(scene, o.runner.last_eval, o.readback_shadow_atlas(w, h))
    f = e.f
    keep = e.shadow_margin > 1e-5
    hdr = o.readback_hdr_f32()
    bad, n, needed = ref.compare(hdr[f.mask], e.want, e.sens, mask=keep, f16=(samples == 4))
    assert n == 4 * np.count_nonzero(keep) and not bad.any(), \
        f"{name}: {bad.sum()} of {n} values outside the bound, first at pixel {np.argwhere(f.mask)[np.argwhere(bad)[0][0]]}"
    clear = np.float32(scenes.CLEAR) if samples == 1 else np.float16(scenes.CLEAR).astype(np.float32)   # 4x: rgba16f samples
    assert np.all(hdr[~f.mask] == clear)
    if name.startswith("grid") or name.startswith("shadow"):
        assert needed < 0.05, f"{needed:.2%} of the values needed the sensitivity allowance"
    if name.startswith("shadow"):
        assert np.count_nonzero(~keep) < 0.02 * len(keep), "too many shadow ties"


@pytest.mark.parametrize("kind", ["negative", "nan"])
def test_degenerate_radius_lights_every_fragment(kind):
    """A negative or NaN radius gives att = 1 at any distance: the oracle shades the whole grid brighter than without that light,
    including fragments far beyond |radius|."""
    scene = scenes.degenerate_light_scene(kind)
    with_light = oracle_frame(scene, 1).readback_hdr_f32()
    scene.point_lights.pop()
    without = oracle_frame(scene, 1).readback_hdr_f32()
    f = scenes.fragments(scene)
    far = f.mask.copy()
    yy, xx = np.mgrid[0:scene.height, 0:scene.width]
    far &= np.hypot(xx + 0.5 - 60.0, yy + 0.5 - 25.0) > 20.0
    brighter = (with_light[..., :3] > without[..., :3]).any(axis=2)
    assert np.count_nonzero(brighter & far) > 0.3 * np.count_nonzero(far)
