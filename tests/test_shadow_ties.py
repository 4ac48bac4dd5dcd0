"""The directional shadow lookup where ties decide it: a two-sided floor that shadows itself (tests/shadow_tie_scenes.py), read back
through the probe material.  On the CPU the float32 restatement (tests/shadow_lookup_reference.py) equals the oracle bit for bit;
on the GPU the shadow factor recovered from every pixel equals the oracle's to 1e-6 at 1x, with no tie left out, with and without a
texture table, and with the lights read from shared and from global memory.  The 4x runs hold the resolved colour only to one
half-precision step, since the samples are rounded to rgba16f before they are compared."""
import numpy as np
import pytest

import shadow_lookup_reference as ref
import shadow_tie_scenes as scenes
from harness import same_bytes
from oracle import load_oracle_backend

SCENES = list(scenes.SCENES)
# the probe's rounding: the kernels' n.l and diffuse term are within a few float32 ulps of the oracle's, so a recovered factor is
# good to about 1e-6; a flipped tap moves it by 0.2 x its bilinear weight, so every flip with a weight of 1e-5 or more shows
RECOVER_TOL = 1e-6


def draw(backend, name, samples, tex=False):
    r = scenes.render(backend, name, samples, tex)
    ev = r.last_eval
    atlas = backend.readback_shadow_atlas(*ev.shadow_target_size).copy()
    return dict(runner=r, atlas=atlas, depth=backend.readback_depth().copy(), hdr=backend.readback_hdr_f32().copy())


def oracle_frame(name, samples=1):
    b = load_oracle_backend()
    b.set_parity_target(True)
    out = draw(b, name, samples)
    out["restated"] = scenes.restate(out["runner"], name, out["atlas"], out["depth"] != 0.0)   # reverse Z: cleared to 0
    b.close()
    return out


def first_failure(rs, bad, got, want, what):
    """The first failing pixel with its light's whole chain, restated."""
    k, c = map(int, np.argwhere(bad)[0])
    ys, xs = np.nonzero(rs.mask)
    i = rs.channel_light[c]
    return (f"{what}: {int(bad.sum())} of {bad.size} lookups differ; first at pixel ({xs[k]}, {ys[k]}), channel {c} = light {i}: got "
            f"{got[k, c]!r}, want {want[k, c]!r}\n{ref.describe(rs.lookups[i], k, i)}")


@pytest.mark.parametrize("name", SCENES)
def test_restatement_equals_oracle_bit_for_bit(name):
    """Every pixel of the probe, every tie included: the restated HDR (factor, n.l and diffuse term in float32) is the oracle's.
    Under the linear sampler the checker's albedo may round below 1, so there the factors are compared, to the probe's rounding."""
    o = oracle_frame(name)
    rs = o["restated"]
    if scenes.SCENES[name].eye is None:
        assert rs.exact.all(), "a pixel centre lies on the floor's diagonal"
    else:
        assert rs.exact.mean() >= 0.97, "too many pixel centres on the floor's edges"
    if scenes.SCENES[name].sampler == "linear":
        got, want = rs.recover(o["hdr"]), rs.factors()
        bad = ~np.isnan(want) & ~(np.abs(got - want) <= 0.25 * RECOVER_TOL)
    else:
        got, want = o["hdr"][rs.mask][:, :3], rs.hdr
        bad = got.view(np.uint32) != want.view(np.uint32)
    bad &= rs.exact[:, None]   # on an edge the raster's tie rule, not restated here, picks the triangle
    assert not bad.any(), first_failure(rs, bad, got, want, f"{name}: restatement vs oracle")


@pytest.mark.parametrize("name", SCENES)
def test_census_reaches_the_ties(name):
    """The scene is in the regime it is meant to test: most lit lookups have a compare within 4 ulps of their reference depth,
    many factors are partial, the atlas width is not a power of two, the tiles are away from the origin, with more than 8 lights
    some probed light is one the kernels read from global memory, the edge scenes wrap taps at the atlas border and put fragments
    between the region test's bound and the tile edge, the checker's holes reach the lookups, the tilted floor uses the x,
    y and z terms of the shadow-space depth, and the exact floor has n.l = 1."""
    fl = scenes.SCENES[name]
    o_frame = oracle_frame(name)
    rs = o_frame["restated"]
    edges = fl.distance == 100.0
    if fl.eye is None:
        assert rs.identity_view
    else:
        assert not rs.identity_view and len(rs.vp) >= 1000, "the look-at floor should cover at least 1000 pixels"
        assert all(np.count_nonzero((lm != 0) & (lm != 1) & (lm != -1)) >= 12 for lm in rs.lm), "light.view_proj * inv_view is trivial"
    covered = rs.mask.sum() / rs.inside.sum()
    if fl.sampler:
        assert 0.3 <= covered <= 0.7, f"the checker leaves {covered:.0%} of the floor"
    else:
        assert covered == 1.0
    probed = [i for i in rs.channel_light if i is not None]
    for i in probed:
        o = rs.lookups[i]
        assert o.sampled.mean() >= (0.5 if edges or fl.eye else 0.9), f"light {i}: only {o.sampled.mean():.2%} of the floor is sampled"
        assert ref.near_ties(o)[o.sampled].mean() >= 0.3, f"light {i}: too few ties"
        partial = (o.factor > 0) & (o.factor < 1)
        assert partial.mean() >= 0.05, f"light {i}: only {partial.mean():.2%} partial factors"
        if fl.sampler:
            holes = np.zeros(len(o.flx), dtype=bool)
            for t in o.texels:
                holes |= (t == 0.0).any(axis=1)
            assert (holes & o.sampled).mean() >= 0.1, "too few lookups reach a hole of the checker in the atlas"
        if fl.slope_x:
            assert all(rs.lm[i][k] != 0 for k in (2, 6, 10)), "a term of the shadow-space depth is 0"
        if name.startswith("exact"):
            assert (rs.nol[i] == 1.0).all()
    atlas_w = int(round(1.0 / float(rs.lights[0]["inv_resolution"][0])))
    if fl.n_lights > 1:
        assert atlas_w & (atlas_w - 1) != 0, f"atlas width {atlas_w} is a power of two"
        assert (rs.lights["atlas_offset"] != 0).any(axis=1).sum() >= fl.n_lights - 1
    if fl.n_lights > 8:
        assert max(probed) >= 8, "no probed light past the shared-memory stage"
    if edges:
        if fl.n_lights == 1:   # the one tile is the whole atlas
            assert sum(int(scenes.wraps(rs.lookups[i], o_frame["atlas"].shape).sum()) for i in probed) >= 100, "no tap wraps at the atlas border"
        assert sum(int(scenes.in_bound_band(rs.lookups[i], rs.lights[i]).sum()) for i in probed) >= 10, "no fragment between the bound and the edge"


# ------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("tex", [False, True], ids=["plain", "texture_table"])
@pytest.mark.parametrize("samples", [1, 4])
@pytest.mark.parametrize("name", SCENES)
def test_gpu_lookup_at_ties(name, samples, tex):
    """Atlas and depth bit for bit; at 1x the factor recovered from each pixel equals the oracle's and the restatement's within the
    probe's rounding (1e-6), and on the exact floor the HDR is the oracle's bit for bit.  At 4x the samples are rounded to
    rgba16f before the resolve, so the resolved colour is only held to the oracle's within one half-precision step (2^-10
    relative): a flipped tap shows there only when 0.2 x its weight exceeds about 1e-3 of the value, far looser than at 1x."""
    from rend3_b200.backend import load_cuda_backend

    o = oracle_frame(name, samples)
    rs = o["restated"]
    b = load_cuda_backend(0, parity_target=True)
    g = draw(b, name, samples, tex)
    b.close()
    assert same_bytes(g["atlas"], o["atlas"]), "shadow atlas differs from the oracle"
    assert same_bytes(g["depth"], o["depth"]), "depth differs from the oracle"
    if samples == 1:
        want = rs.factors()
        got = rs.recover(g["hdr"])
        orc = rs.recover(o["hdr"])
        live = ~np.isnan(want)
        assert np.abs(orc - want)[live].max() <= 0.25 * RECOVER_TOL, "the probe does not recover the oracle's own factors"
        bad = live & ~(np.abs(got - want) <= RECOVER_TOL)
        assert not bad.any(), first_failure(rs, bad, got, want, f"{name}, tex={tex}: GPU vs restatement")
        if name.startswith("exact"):
            got, want = g["hdr"][rs.mask][:, :3], o["hdr"][rs.mask][:, :3]
            bad = got.view(np.uint32) != want.view(np.uint32)
            assert not bad.any(), first_failure(rs, bad, got, want, f"{name}, tex={tex}: GPU HDR vs oracle HDR, bit for bit")
    else:
        got, want = g["hdr"][rs.mask][:, :3], o["hdr"][rs.mask][:, :3]
        bad = ~(np.abs(got - want) <= np.abs(want) * 2.0 ** -10 + 2.0 ** -24)
        assert not bad.any(), f"{int(bad.sum())} resolved values differ from the oracle by more than a half-precision step"
