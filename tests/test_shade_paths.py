"""The shading kernels of rend3_b200/csrc/r3_shade.cu (resolve_kernel<1|4, TEX>, blend_apply_kernel) against the CPU oracle and
the float64 fs_main of tests/shade_reference.py, on the closed-form scenes of tests/shade_scenes.py.

Every scene runs with no texture table and with an unused texture bound, so both resolve_kernel<S, false> and <S, true> shade
untextured materials.  Depth and the shadow atlas are identical to the oracle's.  Pixels are within TOL (relative above 1.0) plus
the reference's sensitivity allowance of the oracle, and within the same bound of the reference, except where a shadow lookup is
decided by 1e-5 or less.  The allowance is needed near the GGX peak, where the kernel's FMA contraction and MUFU approximations are
amplified by 1/a^2 as the oracle's f32 rounding is.  The cases aim at the light-loop edges: the 32-light mask words, the point
lights past the 128 staged in shared memory (never tile-culled), the directional lights past the 8 staged ones with real shadow
maps, the tile-culling box at and around a light's radius, roughness 0 (no culling), and light records with a radius that is 0,
negative, NaN, infinite, or whose square overflows or underflows."""
import numpy as np
import pytest

import shade_reference as ref
import shade_scenes as scenes
from rend3_b200.backend import load_cuda_backend
from shade_reference import TOL

from oracle import load_oracle_backend

pytestmark = pytest.mark.gpu
TIE = 1e-5          # shadow lookups decided by less are left to the oracle comparison


@pytest.fixture()
def cuda():
    b = load_cuda_backend(0, parity_target=True)
    yield b
    b.close()


def atlas(backend, runner):
    w, h = runner.last_eval.shadow_target_size
    return backend.readback_shadow_atlas(w, h)


def f16_bound(v, steps):
    return steps * np.maximum(np.abs(v) * 2.0 ** -10, 2.0 ** -24)


class Case:
    """One scene rendered on the CUDA path and the oracle in every configuration a test asks for, with the float64 reference
    evaluated once (it does not depend on the sample count or the texture table)."""

    def __init__(self, cuda, scene, translucent=None):
        self.cuda, self.scene, self.translucent = cuda, scene, translucent
        self.exp = self.front = None

    def render(self, samples, tex, **kw):
        orc = load_oracle_backend()
        runners = [scenes.render(b, self.scene, samples, texture_table=tex, translucent=self.translucent, **kw) for b in (self.cuda, orc)]
        ac, ao = atlas(self.cuda, runners[0]), atlas(orc, runners[1])
        assert np.array_equal(ac.view(np.uint32), ao.view(np.uint32)), "shadow atlas differs from the oracle"
        if self.exp is None:
            self.exp = scenes.expected(self.scene, runners[0].last_eval, ac)
            if self.translucent is not None:
                self.front = scenes.expected(scenes.translucent_copy(self.scene, self.translucent), runners[0].last_eval, ac)
        return orc

    def want(self, samples):
        """(value, allowance, f16 steps) images of what the target holds: the opaque shade, or one translucent layer blended over
        it by rule R8 in half precision."""
        e = self.exp
        want, sens = e.image(e.want, np.nan), e.image(e.sens)
        steps = 1 if samples == 4 else 0
        if self.front is not None:
            src, src_sens = self.front.image(self.front.want, np.nan), self.front.image(self.front.sens)
            a = src[..., 3:]
            dst = np.float16(want).astype(np.float64)
            want = np.concatenate([src[..., :3] * a + dst[..., :3] * (1.0 - a), a + dst[..., 3:] * (1.0 - a)], axis=-1)
            sens = a * src_sens + (1.0 - a) * sens
            steps = 2
        return want, np.nan_to_num(sens, nan=0.0), steps

    def check(self, samples, what, mask=None, orc=None):
        cuda, e = self.cuda, self.exp
        dc, do = cuda.readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32)
        assert np.array_equal(dc, do), f"{what}: {np.count_nonzero(dc != do)} depth texels differ from the oracle"
        a, o = cuda.readback_hdr_f32().astype(np.float64), orc.readback_hdr_f32().astype(np.float64)
        want, sens, steps = self.want(samples)
        sel = np.ones(e.f.mask.shape, dtype=bool) if mask is None else mask
        bound = TOL * np.maximum(1.0, np.abs(o)) + f16_bound(o, steps) + sens
        bad = ~(np.abs(a - o) <= bound) & sel[..., None]
        assert not bad.any(), f"{what}: {np.count_nonzero(bad)} channel values differ from the oracle beyond the bound " \
                              f"(max excess {np.nanmax(np.abs(a - o) - bound):.3e}), first at {np.argwhere(bad)[0]}"
        keep = sel & e.f.mask & (e.image(e.shadow_margin, np.inf) > TIE)
        if self.front is not None:
            keep &= self.front.image(self.front.shadow_margin, np.inf) > TIE
        bad = (np.abs(a - want) > TOL * np.maximum(1.0, np.abs(want)) + f16_bound(want, steps) + sens) & keep[..., None] & np.isfinite(want)
        n = np.count_nonzero(keep)
        assert n > 0 and not bad.any(), f"{what}: {np.count_nonzero(bad)} values of {n} pixels outside the reference's bound, " \
                                        f"first at {np.argwhere(bad)[0] if bad.any() else None}"
        return a

    def run(self, samples_list=(1, 4), what=""):
        for samples in samples_list:
            for tex in (False, True):
                orc = self.render(samples, tex)
                self.check(samples, f"{what} {samples}x tex={tex}", orc=orc)


def test_material_grid(cuda):
    Case(cuda, scenes.grid_with_lights(40, 3)).run(what="material grid")


def test_material_grid_blended(cuda):
    """A translucent copy of every quad in front of the grid: blend_apply_kernel shades it with the same lights."""
    c = Case(cuda, scenes.grid_with_lights(40, 3), translucent=0.4)
    c.run(what="blended grid")
    assert cuda.forward_stats()[3] > 0


@pytest.mark.parametrize("n_point", [0, 1, 31, 32, 33, 127, 128, 129, 300])
def test_point_light_counts(cuda, n_point):
    """Either side of every 32-light mask word, and past the 128 lights staged in shared memory."""
    scene = scenes.grid_with_lights(n_point, 1, seed=n_point)
    for l in scene.point_lights:
        l.intensity *= 8.0 / max(n_point, 8)        # keep the sum of many lights in the same range
    Case(cuda, scene).run(what=f"{n_point} point lights")


@pytest.mark.parametrize("n_dir", [1, 8, 9, 12])
def test_shadowed_directional_lights(cuda, n_dir):
    """Either side of the 8 directional lights staged in shared memory, each with a real shadow map: occluders over a floor the
    shadow passes cull.  The compared pixels include lit, fully shadowed and fractional-PCF ones, and (over the four light counts)
    the exact-1 cases of fs_main's region test: the any() quirk failing, and shadow depth outside [0, 1]."""
    c = Case(cuda, scenes.shadow_scene(n_dir))
    c.run(what=f"{n_dir} shadowed directional lights")
    e = c.exp
    decided = (e.shadow_margin > TIE)[:, None] & e.sampled
    assert np.count_nonzero(decided & (e.shadow == 1.0)) and np.count_nonzero(decided & (e.shadow == 0.0)), "no lit or no shadowed pixel"
    assert np.count_nonzero(decided & (e.shadow > 0.0) & (e.shadow < 1.0)) > 100, "no fractional PCF pixels"
    assert np.count_nonzero(~e.sampled & (e.shadow_margin > TIE)[:, None]) > 0, "no pixel outside the shadow region"
    assert np.count_nonzero(e.shadow_margin <= TIE) < 0.02 * len(e.shadow_margin), "too many shadow ties"


LAYOUTS = {
    **{f"tangent_{f!r}": (lambda f=f: scenes.tangent_layout(f)) for f in scenes.TANGENT_FACTORS},
    "pythagorean": scenes.pythagorean_layout,
    "far_small_radii": scenes.far_layout,
    "half_covered_tiles": scenes.half_covered_layout,
}
EXACT_COUNT = {"tangent_1.0005", "tangent_1.002", "far_small_radii", "half_covered_tiles"}


@pytest.mark.parametrize("name", list(LAYOUTS))
def test_tile_culling_layouts(cuda, name):
    """Pixel values, and the single-sample light evaluations: within the counts for radii moved by the f32 uncertainty of the view
    position, and exact where no fragment is that close to a radius, so that a light the tile test wrongly drops lowers it."""
    scene = LAYOUTS[name]()
    c = Case(cuda, scene)
    c.run(what=name)
    lo, hi = scenes.light_evaluation_bounds(scene)
    assert lo == hi or name not in EXACT_COUNT
    c.render(1, False)
    assert lo <= cuda.forward_light_evaluations() <= hi, (cuda.forward_light_evaluations(), lo, hi)


def test_scissor_rows(cuda):
    """A second frame shaded only in rows [13, 37) (the row split of the multi-GPU forward pass, begin not a multiple of 8):
    the rows inside equal a full frame of the new lights and the reference, the rows outside keep the first frame.  Once without
    and once with a skybox behind the grid, so that skybox_kernel's rows are scissored too."""
    import skybox_case

    sky_faces = skybox_case.random_faces(16, "rgba8_srgb", seed=13)
    for sky in (False, True):
        scene = scenes.grid_with_lights(40, 1)

        def build(b, scene):
            r = scenes.build(b, scene)
            if sky:
                r.renderer.set_skybox(sky_faces, srgb=True)
            return r

        orc = load_oracle_backend()
        runners = {id(b): build(b, scene) for b in (cuda, orc)}
        for b in (cuda, orc):
            scenes.draw(runners[id(b)], scene, 1)
        first = cuda.readback_hdr_f32()
        moved = scenes.grid_with_lights(40, 1)
        moved.point_lights = scenes.random_point_lights(40, seed=7)
        for b in (cuda, orc):
            runners[id(b)].renderer.point_lights = moved.point_lights
            scenes.draw(runners[id(b)], scene, 1, scissor_rows=(13, 37))
        inside = np.zeros((scene.height, scene.width), dtype=bool)
        inside[13:37] = True
        c = Case(cuda, moved)
        c.exp = scenes.expected(moved, runners[id(cuda)].last_eval, atlas(cuda, runners[id(cuda)]))
        a = c.check(1, f"scissored frame, sky {sky}", mask=inside, orc=orc)
        assert np.array_equal(a[~inside], first[~inside].astype(np.float64)), "rows outside the scissor were written"
        fresh = load_cuda_backend(0, parity_target=True)
        scenes.draw(build(fresh, moved), moved, 1)
        assert np.array_equal(a[inside], fresh.readback_hdr_f32()[inside].astype(np.float64)), "rows inside differ from the full frame"
        fresh.close()
        if sky:
            import skybox_reference

            sky_px = inside & ~c.exp.f.mask
            assert np.count_nonzero(sky_px) > 100, "no sky inside the rows"
            skybox_reference.compare(a, skybox_case.reference(runners[id(cuda)], (scene.width, scene.height)), "scissored sky", mask=sky_px)


def peak_mask(scene):
    """Pixels where the GGX denominator 1 - noh^2 (1 - a^2) exceeds 1e-3 for every point light: elsewhere D of a roughness-0
    material is a 0 / 0 or huge."""
    f = scenes.fragments(scene)
    pl_pos, _, _ = scenes.light_arrays(scene)
    margin = np.full((scene.height, scene.width), -1.0)
    margin[f.mask] = ref.ggx_peak_margin(f.vp, f.normal, f.mat, pl_pos)
    return (margin > 1e-3) | ~f.mask


@pytest.mark.parametrize("case", ["roughness_0", "perceptual_1e-10", "clear_coat_to_zero"])
def test_roughness_edges(cuda, case):
    """Roughness 0 takes the unculled path: at the GGX peak its D is 0 * inf = NaN, which the per-light max(s, 0) and the final
    max(ambient * albedo, colour) (minNum / maxNum) remove, so no pixel may be NaN, and the values elsewhere equal the reference.
    Perceptual roughness 1e-10 keeps the tile culling on while a^2 is subnormal; a clear coat of -1 over roughness 0.5 with
    clear-coat roughness 1 drives the perceptual roughness to exactly 0."""
    if case == "roughness_0":
        scene = scenes.grid_with_lights(40, 1, roughness=0.0)
    elif case == "perceptual_1e-10":
        scene = scenes.grid_with_lights(40, 1, seed=5, roughness=1e-10)
    else:
        scene = scenes.grid_with_lights(40, 1, seed=5, roughness=0.5)
        for q in scene.quads[::3]:
            q.material.clearcoat_factor, q.material.clearcoat_roughness_factor = -1.0, 1.0
    c = Case(cuda, scene)
    for samples in (1, 4):
        for tex in (False, True):
            orc = c.render(samples, tex)
            assert not np.isnan(cuda.readback_hdr_f32()).any() and not np.isnan(orc.readback_hdr_f32()).any()
            c.check(samples, f"{case} {samples}x tex={tex}", mask=peak_mask(scene), orc=orc)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_light_evaluations_count(cuda, seed):
    """With conservative culling a single-sample fragment evaluates every directional light and exactly the point lights with
    d^2 < r^2: the tile test may keep more, the per-fragment test removes them.  A light wrongly dropped by a tile lowers the
    count.  On a roughness-0 grid nothing is skipped: n_dir + n_point per lit fragment."""
    scene = scenes.untie_radii(scenes.grid_with_lights(150, 2, seed=seed))
    lo, hi = scenes.light_evaluation_bounds(scene)
    assert lo == hi, "no fragment may sit within f32 rounding of a radius"
    scenes.render(cuda, scene, 1)
    assert cuda.forward_light_evaluations() == lo
    mirror = scenes.grid_with_lights(150, 2, seed=seed, roughness=0.0)
    for q in mirror.quads:
        q.material.clearcoat_factor = 0.0                 # a clear coat would raise the roughness above 0
    scenes.render(cuda, mirror, 1)
    n_lit = np.count_nonzero(scenes.fragments(mirror).mask)
    assert cuda.forward_light_evaluations() == n_lit * (2 + 150) == scenes.light_evaluations(mirror)


@pytest.mark.parametrize("mode", ["1x", "4x", "blend"])
@pytest.mark.parametrize("kind", scenes.DEGENERATE_KINDS)
def test_degenerate_light_records(cuda, kind, mode):
    """A point light whose radius is 0, negative, NaN, +inf, 1e20 (r^2 overflows) or 1e-23 (r^2 underflows), one of colour 0, and
    one exactly on a fragment's view position.  A negative or NaN radius lights every fragment (saturate(d / r) = 0), on every
    path, so neither the tile test nor the per-fragment test may drop it."""
    scene = scenes.degenerate_light_scene(kind)
    c = Case(cuda, scene, translucent=0.4 if mode == "blend" else None)
    c.run(samples_list=(4,) if mode == "4x" else (1,), what=f"{kind} light" + (" blend" if mode == "blend" else ""))
    if mode == "1x" and kind != "at_fragment":
        c.render(1, False)
        lo, hi = scenes.light_evaluation_bounds(scene)
        assert lo == hi and cuda.forward_light_evaluations() == lo
