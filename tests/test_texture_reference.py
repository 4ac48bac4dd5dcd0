"""Textured shading against the float64 textureSampleGrad and get_pixel_data_inner of tests/texture_reference.py, on the scenes of
tests/texture_scenes.py: the CPU oracle without a GPU, and on the GPU resolve_kernel<1|4, TEX>, blend_apply_kernel and the cutout
discards of the rasteriser (forward pass and shadow pass).

The bound is TOL (relative above 1.0) plus shade_reference's sensitivity allowance plus the sampling bound carried through fs_main
(each sampled channel moved by its bound, either sign), plus the rgba16f rounding at 4x.  Pixels the reference flags (a nearest-
sampler tie, a discard within its bound of the threshold, a non-finite texel the f32 error leaves open) are left out, counted and
capped per scene by FLAG_CAP.  A census per scene asserts that the edges it is built for are reached on compared pixels."""
import functools

import numpy as np
import pytest

import texture_reference as tref
import texture_scenes as ts
from blend_reference import f16
from rend3_b200.layouts import TEXFMT_R8_UNORM, TEXFMT_RGBA8_UNORM, TEXFMT_RGBA8_UNORM_SRGB, TEXTURE_DESC_DTYPE

from oracle import load_oracle_backend

OPAQUE_SCENES = ["levels", "materials", "cutout", "floor"]
# flagged pixels allowed per scene: the nearest quad built at the tie itself (one cell), the texel of the cutout texture that
# sits exactly at the threshold and the cutout edges that fall within the bound, the floor's few pixels at k + 0.5
FLAG_CAP = {"levels": 1100, "materials": 0, "cutout": 400, "floor": 64, "blend": 0}


def atlas(backend, runner):
    w, h = runner.last_eval.shadow_target_size
    return backend.readback_shadow_atlas(w, h)


@functools.lru_cache(maxsize=None)
def oracle_case(name, samples):
    scene = ts.SCENES[name]()
    o = load_oracle_backend()
    r = ts.render(o, scene, samples)
    which = [k for k, q in enumerate(scene.objects) if q.label != "blend"]
    return scene, o, r, ts.expected(scene, o, r, samples, which)


# ------------------------------------------------------------------ the reference itself
def _one(fmt, w, h, levels_bytes):
    d = np.zeros(1, dtype=TEXTURE_DESC_DTYPE)
    d["width"], d["height"], d["mip_count"], d["format"] = w, h, len(levels_bytes), fmt
    return d[0], np.concatenate([np.asarray(b, dtype=np.uint8).reshape(-1) for b in levels_bytes])


def _sample(levels, linear, u, v, du, dv):
    n = len(u)
    z = np.zeros(n)
    return tref.sample_grad(levels, linear, np.asarray(u, float), np.asarray(v, float), np.full(n, du), z, z, np.full(n, dv), z, z)


def test_reference_known_answers():
    g = np.random.default_rng(3)
    l0, l1, l2 = g.integers(0, 256, (4, 8, 4), dtype=np.uint8), g.integers(0, 256, (2, 4, 4), dtype=np.uint8), g.integers(0, 256, (1, 2, 4), dtype=np.uint8)
    d, blob = _one(TEXFMT_RGBA8_UNORM, 8, 4, [l0, l1, l2])
    lv = tref.texture_levels(d, blob)
    assert [x.shape for x in lv] == [(4, 8, 4), (2, 4, 4), (1, 2, 4)]
    t0 = l0.astype(float) / 255
    # texel centres return the texel; one texel per pixel is level 0
    s = _sample(lv, True, [2.5 / 8, 7.5 / 8], [1.5 / 4, 3.5 / 4], 1 / 8, 1 / 4)
    assert np.allclose(s.value, [t0[1, 2], t0[3, 7]], atol=1e-15) and (s.lam == 0).all()
    # Repeat: texel -1 is texel w - 1 and texel w is texel 0, on both sides of the texture
    s = _sample(lv, False, [-0.5 / 8, 8.5 / 8, -7.5 / 8], [0.5 / 4, -0.5 / 4, 4.5 / 4], 1 / 8, 1 / 4)
    assert np.allclose(s.value, [t0[0, 7], t0[3, 0], t0[0, 0]], atol=1e-15)
    s = _sample(lv, True, [0.0], [0.5 / 4], 1 / 8, 1 / 4)                 # halfway between texel 7 (wrapped) and texel 0
    assert np.allclose(s.value, [(t0[0, 7] + t0[0, 0]) / 2], atol=1e-15)
    # exactly 2 texels per pixel: lambda = 1, fraction 0, level 1 alone
    s = _sample(lv, True, [0.3], [0.6], 2 / 8, 0.0)
    assert s.lam[0] == 1.0 and s.fr[0] == 0.0 and np.allclose(s.value, tref.bilinear(lv[1], np.array([0.3]), np.array([0.6])), atol=1e-15)
    # lambda 1.5 blends levels 1 and 2 half and half; past the last level the last level alone; lambda <= 0 is level 0
    s = _sample(lv, True, [0.3], [0.6], 2 ** 1.5 / 8, 0.0)
    want = (tref.bilinear(lv[1], np.array([0.3]), np.array([0.6])) + tref.bilinear(lv[2], np.array([0.3]), np.array([0.6]))) / 2
    assert abs(s.lam[0] - 1.5) < 1e-15 and np.allclose(s.value, want, atol=1e-12)
    s = _sample(lv, True, [0.3], [0.6], 40 / 8, 0.0)
    assert s.level[0] == 2 and np.allclose(s.value, tref.bilinear(lv[2], np.array([0.3]), np.array([0.6])), atol=1e-15)
    # nearest: level floor(lambda + 0.5) on both sides of 1.5, texel floor(u w)
    for rho, level in ((2 ** 1.49, 1), (2 ** 1.51, 2), (2 ** 0.49, 0), (2 ** 0.51, 1)):
        s = _sample(lv, False, [0.3], [0.6], rho / 8, 0.0)
        assert s.level[0] == level and np.array_equal(s.value, tref.nearest(lv[level], np.array([0.3]), np.array([0.6])))
    # the larger of the two derivative lengths decides (anisotropic footprint)
    s = tref.sample_grad(lv, True, np.array([0.3]), np.array([0.6]), np.array([1 / 8]), np.array([0.0]), np.array([0.0]), np.array([4 / 4]),
                         np.zeros(1), np.zeros(1))
    assert s.lam[0] == 2.0
    # sRGB is decoded per texel, before the filter
    d, blob = _one(TEXFMT_RGBA8_UNORM_SRGB, 2, 1, [np.array([[[0, 0, 0, 0], [255, 128, 10, 255]]], np.uint8)])
    lv = tref.texture_levels(d, blob)
    s = _sample(lv, True, [0.5], [0.5], 0.5, 1.0)
    dec = tref.srgb_decode(np.array([1.0, 128 / 255, 10 / 255]))
    assert np.allclose(s.value[0], list(dec / 2) + [0.5], atol=1e-15)
    # missing channels read (0, 0, 1); a slot past the table reads zeros
    d, blob = _one(TEXFMT_R8_UNORM, 2, 2, [np.array([[10, 20], [30, 40]], np.uint8)])
    assert np.allclose(tref.texture_levels(d, blob)[0][1, 0], [30 / 255, 0, 0, 1])
    table = tref.Table(np.array([d]), blob)
    assert table.levels(2) is None and table.levels(1) is not None


# ------------------------------------------------------------------ the oracle
@pytest.mark.parametrize("samples", [1, 4])
@pytest.mark.parametrize("name", OPAQUE_SCENES + ["blend"])
def test_oracle_matches_texture_reference(name, samples):
    scene, o, r, e = oracle_case(name, samples)
    got = o.readback_hdr_f32()
    keep = uncovered_by_blend(scene, o, r, samples) if name == "blend" else None    # the blended quad: test_oracle_blend
    bad, n = ts.compare(got, e, keep)
    assert n > 10000 and not bad.any(), f"{name} {samples}x: {bad.any(-1).sum()} pixels outside the bound, first at {np.argwhere(bad)[0]}"
    assert np.count_nonzero(e.flagged) <= FLAG_CAP[name], f"{np.count_nonzero(e.flagged)} flagged pixels"
    if name == "cutout":
        fwd = e.keep & (e.label != "")
        assert np.array_equal(o.readback_depth()[fwd] == 0, e.discard[fwd]), "the forward discards differ from the reference"
        check_shadow_discards(scene, o, r, atlas(o, r))


def uncovered_by_blend(scene, backend, runner, samples):
    """Pixels the translucent quad leaves alone: there the opaque pass alone decides the target."""
    front = ts.expected(scene, backend, runner, samples, [[q.label for q in scene.objects].index("blend")])
    return (front.label == "") & (front.keep | front.flagged)


def check_shadow_discards(scene, backend, runner, at):
    """Every shadow-atlas texel whose owner is decided and not near its threshold: written exactly where the depth pass keeps it."""
    n = 0
    for region, label, disc, near, decided in ts.shadow_decisions(scene, backend, runner):
        a = at[region]
        m = (label != "") & decided & ~near
        empty = a == a[label == ""][0] if (label == "").any() else np.zeros_like(a, bool)
        assert np.count_nonzero(m & disc) > 100 and np.count_nonzero(m & ~disc) > 100
        bad = m & (empty != disc)
        assert not bad.any(), f"{np.count_nonzero(bad)} shadow texels differ from the depth-pass reference, first at {np.argwhere(bad)[0]}"
        n += np.count_nonzero(m)
    assert n > 300


def blend_expected(scene, backend, runner):
    """The translucent quad over the opaque one and over the clear colour, 1x: src * a + f16(dst) * (1 - a) (rule R8)."""
    idx = [q.label for q in scene.objects]
    back = ts.expected(scene, backend, runner, 1, [idx.index("opaque")])
    front = ts.expected(scene, backend, runner, 1, [idx.index("blend")])
    a = front.want[..., 3:]
    dst = f16(back.want).astype(np.float64)
    want = np.concatenate([front.want[..., :3] * a + dst[..., :3] * (1 - a), a + dst[..., 3:] * (1 - a)], axis=-1)
    bound = a * front.bound + (1 - a) * back.bound + 2 * np.maximum(np.abs(want) * 2.0 ** -10, 2.0 ** -24)
    keep = front.keep & (front.label == "blend") & back.keep
    return want, bound, keep, back.label == "opaque"


def test_oracle_blend():
    scene = ts.SCENES["blend"]()
    o = load_oracle_backend()
    r = ts.render(o, scene, 1)
    want, bound, keep, over = blend_expected(scene, o, r)
    got = o.readback_hdr_f32()
    bad = keep[..., None] & ~(np.abs(got - want) <= bound)
    assert np.count_nonzero(keep & over) > 500 and np.count_nonzero(keep & ~over) > 500
    assert not bad.any(), f"{bad.any(-1).sum()} blended pixels outside the bound, first at {np.argwhere(bad)[0]}"


CENSUS = {
    "levels": dict(fr0=2000, tie_lo=200, tie_hi=200, past_last=500, magnified=2000, aniso=500, negative=1000),
    "floor": dict(tie_lo=40, tie_hi=40, past_last=30, magnified=1000, aniso=1000),
    "cutout": dict(negative=500),
    "materials": dict(),
    "blend": dict(),
}


@pytest.mark.parametrize("name", OPAQUE_SCENES)
def test_scene_census(name):
    """Each scene reaches the edges it is built for on compared pixels, and every quad keeps most of its pixels."""
    for samples in (1, 4):
        scene, o, r, e = oracle_case(name, samples)
        for k, need in CENSUS[name].items():
            assert np.count_nonzero(e.census[k]) >= need, f"{samples}x: {k}: {np.count_nonzero(e.census[k])} < {need}"
        for q in scene.objects:
            if name != "floor" and q.label != "tie_0_0":       # the quad built at the tie itself is flagged as a whole
                assert np.count_nonzero(e.keep & (e.label == q.label)) >= 600, f"{q.label} keeps too few pixels"
        if name == "cutout":
            assert np.count_nonzero(e.discard) > 500 and np.count_nonzero(e.keep & (e.label != "") & ~e.discard) > 500
            for lab in ("transformed", "mirrored", "nearest", "vertex_alpha"):
                m = e.keep & (e.label == lab)
                assert np.count_nonzero(m & e.discard) > 20 and np.count_nonzero(m & ~e.discard) > 20, lab


# ------------------------------------------------------------------ the kernels
@pytest.fixture()
def cuda():
    from rend3_b200.backend import load_cuda_backend
    b = load_cuda_backend(0, parity_target=True)
    yield b
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("samples", [1, 4])
@pytest.mark.parametrize("name", OPAQUE_SCENES + ["blend"])
def test_kernel_matches_texture_reference(cuda, name, samples):
    """resolve_kernel<samples, TEX> (and blend_apply_kernel): depth and the shadow atlas bit-identical to the oracle, every compared
    pixel within the reference's bound, forward and shadow-pass discards as the reference decides them."""
    scene = ts.SCENES[name]()
    rc = ts.render(cuda, scene, samples)
    o = load_oracle_backend()
    ro = ts.render(o, scene, samples)
    ac, ao = atlas(cuda, rc), atlas(o, ro)
    assert np.array_equal(ac.view(np.uint32), ao.view(np.uint32)), "shadow atlas differs from the oracle"
    dc, do = cuda.readback_depth(), o.readback_depth()
    assert np.array_equal(dc.view(np.uint32), do.view(np.uint32)), f"{np.count_nonzero(dc != do)} depth texels differ from the oracle"
    which = [k for k, q in enumerate(scene.objects) if q.label != "blend"]
    e = ts.expected(scene, cuda, rc, samples, which)
    got = cuda.readback_hdr_f32().astype(np.float64)
    keep = uncovered_by_blend(scene, cuda, rc, samples) if name == "blend" else None
    bad, n = ts.compare(got, e, keep)
    print(f"{name} {samples}x: {n} values, {np.count_nonzero(e.flagged)} flagged pixels")
    assert n > 10000 and not bad.any(), f"{bad.any(-1).sum()} pixels outside the reference's bound, first at {np.argwhere(bad)[0]}: " \
                                        f"got {got[tuple(np.argwhere(bad)[0][:2])]}, want {e.want[tuple(np.argwhere(bad)[0][:2])]}"
    assert np.count_nonzero(e.flagged) <= FLAG_CAP[name]
    if name == "cutout":
        fwd = e.keep & (e.label != "")
        assert np.array_equal(dc[fwd] == 0, e.discard[fwd]), "the forward discards differ from the reference"
        check_shadow_discards(scene, cuda, rc, ac)
    if name == "blend" and samples == 1:
        assert cuda.forward_stats()[3] > 0
        want, bound, keep, over = blend_expected(scene, cuda, rc)
        bad = keep[..., None] & ~(np.abs(got - want) <= bound)
        assert np.count_nonzero(keep & over) > 500 and not bad.any(), f"{bad.any(-1).sum()} blended pixels outside the bound"
