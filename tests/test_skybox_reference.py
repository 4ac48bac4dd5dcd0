"""The skybox (skybox.wgsl + rule R10) against the float64 restatement of tests/skybox_reference.py.

The CPU tier checks the oracle, the GPU tier the CUDA path (its f32 parity target and its rgba16f target) and its agreement with the
oracle, on the scenes of tests/skybox_case.py: the six axis views of a labelled cube in both handednesses, random views with roll at
FOVs from 2 to 179 degrees (orthographic and raw projections, odd non-square targets, faces 1 to 256 wide, RGBA8, RGBA8 sRGB and
RGBA32F with infinities and NaN, generated mips or none), exact face ties, camera positions, faces at a byte offset, the passes
that draw the sky (resolve at one and four samples, the blend under a translucent cube), and graph-submitted frames.

Error bound (derived in skybox_reference.Sky.bound_of): away from face ties the sample is continuous in (s, t) and lambda — bilinear
weights are continuous, trilinear filtering is continuous at integer lambda, at lambda <= 0 and at the clamp to the last level — so

    |x - ref| <= 1e-4 max(1, |ref|) + R (w_level (eps_st + 4u) + eps_lam) + 8u A

with R the texel range over every footprint the f32 path can fetch, w_level the finest level's width, eps_st the bound on the f32
error of (s, t) derived per pixel from the operations that produce it (about 2^-21 for an ordinary view), eps_lam rule R9's log2
error (< 4e-7) plus the error of rho, which the f32 forward differences carry, A the largest |texel| (the f32 lerps' roundings), and
1e-4 max(1, |ref|) the decode of a texel (sRGB's powf, 1/255).  Where the two largest |components| of the direction differ by less
than their f32 errors the face is not decided: such a flagged pixel passes if it matches either candidate face's value.  A
constructed exact tie is not flagged — the rule decides it.  A value of the rgba16f target must lie in [f16(ref - b), f16(ref + b)]:
f16 rounding is monotonic, so it is within one half-precision step of the bound and overflows to infinity past 65504."""
import dataclasses

import numpy as np
import pytest

import skybox_case as sk
import skybox_reference as sref
from rend3_b200.backend import R3Error
from rend3_b200.layouts import TEXFMT_RGBA32_FLOAT
from rend3_b200.world import LEFT, RIGHT, Renderer

from oracle import load_oracle_backend

f32 = np.float32
U = 2.0 ** -24


@pytest.fixture(params=["oracle", pytest.param("cuda", marks=pytest.mark.gpu)])
def side(request):
    """The backend under test: the oracle on the CPU tier, the CUDA path (parity target on) on the GPU tier."""
    if request.param == "oracle":
        yield request.param, load_oracle_backend
        return
    from rend3_b200.backend import load_cuda_backend

    made = []

    def make():
        made.append(load_cuda_backend(0, parity_target=True))
        return made[-1]

    yield request.param, make
    for b in made:
        b.close()


def f16(v):
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(v, dtype=np.float64).astype(np.float16).astype(np.float64)


def compare_f16(got, sky: sref.Sky, what):
    """The rgba16f target: [f16(ref - b), f16(ref + b)] for either accepted face; non-finite values as in sref.compare."""
    got = np.asarray(got, dtype=np.float64)
    oks = []
    for smp, b in zip((sky.main, sky.alt), sky.bounds()):
        ref, nf = smp.value, smp.nonfinite
        with np.errstate(invalid="ignore"):
            fin = (f16(ref - b) <= got) & (got <= f16(ref + b))
            nonfin = (np.isnan(got) == np.isnan(ref)) & (np.isnan(ref) | (got == ref) | fin)
        open_ = nf.any(-1) & smp.moved
        oks.append(np.where(nf, nonfin, fin).all(-1) | open_)
    ok = oks[0] | (sky.flagged & oks[1])
    assert ok.all(), f"{what}: {np.count_nonzero(~ok)} rgba16f pixels outside [f16(ref - b), f16(ref + b)], first at {np.argwhere(~ok)[0]}"


RATIOS = {}


def check(b, sky: sref.Sky, what, samples=1, orc=None):
    """The backend's f32 target against the reference (at four samples it holds the f16 sky), its rgba16f target on CUDA, and CUDA
    against the oracle: NaN on the same pixels, the other values within 1e-5 relative plus the roundings of the lerps."""
    got = b.readback_hdr_f32()
    if samples == 1:
        c = sref.compare(got, sky, what)
        RATIOS[what] = c
    else:
        compare_f16(got, sky, what + " (4x resolve)")
    if orc is not None:
        compare_f16(b.readback_hdr_f16().astype(np.float64), sky, what + " rgba16f")
        o = orc.readback_hdr_f32().astype(np.float64)
        a = got.astype(np.float64)
        assert np.array_equal(np.isnan(a), np.isnan(o)), f"{what}: NaN on {np.count_nonzero(np.isnan(a) != np.isnan(o))} other pixels than the oracle's"
        fin = np.isfinite(o)
        assert np.array_equal(a[~fin & ~np.isnan(o)], o[~fin & ~np.isnan(o)]), f"{what}: infinities differ from the oracle"
        tol = 1e-5 * np.maximum(1.0, np.abs(o)) + 16 * U * np.where(np.isfinite(sky.main.big), sky.main.big, 0.0)
        with np.errstate(invalid="ignore"):
            bad = fin & ~(np.abs(a - o) <= tol)
        assert not bad.any(), f"{what}: {np.count_nonzero(bad)} values differ from the oracle, first at {np.argwhere(bad)[0]}"
    return got


def render_both(kind, make, v, samples=1):
    """Render `v` on the backend under test (and on the oracle too when that is CUDA); return (backend, oracle or None, reference)."""
    b = make()
    _, sky = sk.render(b, v, samples)
    orc = None
    if kind == "cuda":
        orc = load_oracle_backend()
        sk.render(orc, v, samples)
    return b, orc, sky


# ------------------------------------------------------------------ a. orientation
@pytest.mark.parametrize("handedness", [LEFT, RIGHT])
def test_face_orientation(side, handedness):
    """Each axis view of the labelled cube at one texel per pixel reads its own face, texel (px, py) in a left-handed world — the
    Vulkan table puts s along the view's right and t along its down — and the mirror image (n - 1 - px, py) in a right-handed one,
    whose view's right is the other way round.  The reference states the same and the backend matches the reference."""
    kind, make = side
    n = 16
    faces = sk.labelled_faces(n)
    py, px = np.mgrid[0:n, 0:n]
    col = px if handedness == LEFT else n - 1 - px
    for f in range(6):
        v = sk.SkyView(faces, mips="none", view=sk.axis_view(f, handedness), projection=("perspective", 90.0, 0.1), resolution=(n, n),
                       handedness=handedness)
        b, orc, sky = render_both(kind, make, v)
        want = np.stack([col, py, np.full_like(px, f), np.ones_like(px)], axis=-1).astype(np.float64)
        assert np.all(sky.face == f) and not sky.flagged.any()
        assert np.abs(sky.value - want).max() < 1e-3, f"reference: face {f} {handedness} is not oriented as the Vulkan table says"
        got = check(b, sky, f"orientation face {f} {handedness} {kind}", orc=orc)
        assert np.array_equal(np.rint(got), want), f"face {f} {handedness}: a pixel read another texel"


# ------------------------------------------------------------------ b. random views
def random_views():
    """(name, SkyView) over the FOVs, projections, targets, face widths, mip modes and formats of the issue's scene list."""
    out = []
    cases = [
        ("fov2_w256_srgb", ("perspective", 2.0, 0.1), (97, 61), 256, "generated", "rgba8_srgb"),
        ("fov60_w64_rgba8", ("perspective", 60.0, 0.1), (97, 61), 64, "generated", "rgba8"),
        ("fov90_w5_f32", ("perspective", 90.0, 0.1), (61, 97), 5, "generated", "rgba32f"),
        ("fov150_w3_f32_none", ("perspective", 150.0, 0.1), (97, 61), 3, "none", "rgba32f"),
        ("fov150_w1_srgb", ("perspective", 150.0, 0.1), (97, 61), 1, "generated", "rgba8_srgb"),
        ("fov150_w3_tiny_target", ("perspective", 150.0, 0.1), (7, 5), 3, "generated", "rgba32f"),
        ("ortho_w64_f32", ("orthographic", (6.0, 4.0, 2.0)), (33, 21), 64, "generated", "rgba32f"),
        ("raw_offaxis_w256_rgba8_none", ("raw", sk.offaxis_projection(70.0, 97 / 61)), (97, 61), 256, "none", "rgba8"),
        ("fov120_w256_f32", ("perspective", 120.0, 0.1), (97, 61), 256, "generated", "rgba32f"),
        ("fov179_w8_f32", ("perspective", 179.0, 0.1), (97, 61), 8, "generated", "rgba32f"),
    ]
    for i, (name, proj, res, w, mips, fmt) in enumerate(cases):
        faces = sk.random_faces(w, fmt, seed=100 + i)
        out.append((name, sk.SkyView(faces, srgb=fmt == "rgba8_srgb", mips=mips, view=sk.random_rotation(200 + i), projection=proj, resolution=res)))
    return out


def test_random_views(side):
    """Every scene within the bound; together they reach lambda <= 0, 0 < lambda < last, lambda > last, all six faces and pixels
    next to seams, and NaN texels land on the same pixels as the reference's."""
    kind, make = side
    lam_le0 = lam_mid = lam_above = 0
    faces_seen, seams, nan_pixels, n_flagged = set(), 0, 0, 0
    for name, v in random_views():
        b, orc, sky = render_both(kind, make, v)
        got = check(b, sky, f"{name} {kind}", orc=orc)
        lam = sky.main.lam
        lam_le0 += np.count_nonzero(lam <= 0)
        if sky.last >= 1:
            lam_mid += np.count_nonzero((lam > 0) & (lam < sky.last))
            lam_above += np.count_nonzero(lam > sky.last)
        faces_seen |= set(np.unique(sky.face).tolist())
        seams += np.count_nonzero(sky.seam)
        nan_pixels += np.count_nonzero(np.isnan(got).any(-1))
        n_flagged += np.count_nonzero(sky.flagged)
        assert np.count_nonzero(sky.flagged) <= 0.002 * sky.face.size + 2, f"{name}: {np.count_nonzero(sky.flagged)} face-tie pixels"
    assert lam_le0 > 100 and lam_mid > 100 and lam_above >= 6, (lam_le0, lam_mid, lam_above)
    assert faces_seen == set(range(6)) and seams > 100 and nan_pixels > 10, (faces_seen, seams, nan_pixels)
    worst = max(RATIOS[f"{name} {kind}"].worst_ratio for name, _ in random_views())
    print(f"\nrandom views on {kind}: worst error / bound {worst:.3g}, "
          f"{n_flagged} flagged face-tie pixels")


# ------------------------------------------------------------------ c. exact ties
TIE_VIEWS = sk.TIE_VIEWS
TIE_AXES = {"x_y": (0, 1), "x_z": (0, 2), "y_z": (1, 2), "x_y_back": (0, 1)}


@pytest.mark.parametrize("name", list(TIE_VIEWS))
def test_exact_face_ties(side, name):
    """Permutation views on a 64 x 64 target at 130 degrees: on both diagonals cy = -cx exactly, so two |components| are equal bit
    for bit in f32 and f64; where they are the major axis the rule picks X over Y and Y over Z."""
    kind, make = side
    n = 64
    v = sk.SkyView(sk.labelled_faces(8), view=sk.permutation_view(TIE_VIEWS[name]), projection=("perspective", 130.0, 0.1), resolution=(n, n))
    b, orc, sky = render_both(kind, make, v)
    py, px = np.mgrid[0:n, 0:n]
    diag = (px == py) | (px + py == n - 1)
    ties = sky.exact_tie
    assert np.array_equal(ties & diag, ties), "a tie off the diagonals"
    a, c = TIE_AXES[name]
    tied_major = ties & np.isin(sky.face // 2, (a, c))
    assert np.count_nonzero(tied_major) >= 40, f"only {np.count_nonzero(tied_major)} exact ties of the major axes"
    assert np.all(sky.face[tied_major] // 2 == a), "the reference breaks the tie the wrong way"
    got = check(b, sky, f"ties {name} {kind}", orc=orc)
    assert np.array_equal(np.rint(got[..., 2][tied_major]), sky.face[tied_major]), f"{name}: a tie went to the wrong face"


# ------------------------------------------------------------------ d. camera position
def test_camera_position_does_not_move_the_sky(side):
    """The same rotation at three camera positions: orig_view drops the translation, so the sky is identical bit for bit."""
    kind, make = side
    rot = sk.random_rotation(7)
    images = []
    for t in [(0.0, 0.0, 0.0), (1e3, -250.5, 3.25), (-0.125, 7e4, -9e3)]:
        view = rot.copy()
        view[3, :3] = t
        v = sk.SkyView(sk.random_faces(32, "rgba8_srgb", 3), srgb=True, view=view, projection=("perspective", 75.0, 0.1), resolution=(64, 48))
        b, orc, sky = render_both(kind, make, v)
        images.append(check(b, sky, f"position {t} {kind}", orc=orc).view(np.uint32))
    assert all(np.array_equal(images[0], im) for im in images[1:])


# ------------------------------------------------------------------ e. byte offset
@pytest.mark.parametrize("fmt", ["rgba8", "rgba32f"])
def test_faces_at_a_byte_offset(side, fmt):
    """The faces at byte_offset 16 and 48 of a padded blob, set through the backend, give the image of offset 0 bit for bit; a blob
    one byte short is R3_E_INVALID."""
    kind, make = side
    v = sk.SkyView(sk.random_faces(16, fmt, 11), view=sk.random_rotation(12), projection=("perspective", 100.0, 0.1), resolution=(40, 30))
    b = make()
    r = sk.runner(b, v)
    ev = sk.draw(r, v.resolution)
    first = b.readback_hdr_f32()
    sref.compare(first, sk.reference(r, v.resolution), f"offset 0 {fmt} {kind}")
    first = first.view(np.uint32).copy()
    blob = ev.skybox_texels
    for off in (16, 48):
        rng = np.random.default_rng(off)
        padded = np.concatenate([rng.integers(0, 256, off, dtype=np.uint8), blob, rng.integers(0, 256, 32, dtype=np.uint8)])
        desc = ev.skybox_desc.copy()
        desc["byte_offset"] = off
        b.set_skybox(desc, padded)
        sk.draw(r, v.resolution, upload=False)
        assert np.array_equal(b.readback_hdr_f32().view(np.uint32), first), f"offset {off}"
        with pytest.raises(R3Error) as e:
            b.set_skybox(desc, padded[:off + len(blob) - 1])
        assert e.value.code == -1
    assert int(ev.skybox_desc["format"]) == (TEXFMT_RGBA32_FLOAT if fmt == "rgba32f" else 0)


# ------------------------------------------------------------------ f. every pass that draws the sky
@pytest.mark.parametrize("samples", [1, 4])
def test_sky_passes(side, samples):
    """With no geometry every pixel holds the f16 reference sky.  Under an unlit translucent cube (alpha 0.5) the covered pixels hold
    rule R8 over the f16 sky: skybox_kernel then the blend at one sample, the blend's own re-shade of the sky at four.  A 4x pixel
    the cube covers in part lies between its sky and its blended value."""
    kind, make = side
    v = sk.SkyView(sk.random_faces(32, "rgba32f", 21), view=sk.random_rotation(22), projection=("perspective", 80.0, 0.1), resolution=(72, 56))
    b, orc, sky = render_both(kind, make, v, samples)
    if kind == "cuda":
        compare_f16(b.readback_hdr_f16().astype(np.float64), sky, f"empty {samples}x rgba16f")
    compare_f16(f16(b.readback_hdr_f32()), sky, f"empty {samples}x")
    ok_sky = ~sky.flagged & ~(sky.main.nonfinite.any(-1))
    backends = [b] + ([orc] if orc is not None else [])
    outs = []
    for x in backends:
        r = sk.runner(x, v)
        src = sk.translucent_cube(r, v.view)
        sk.draw(r, v.resolution, samples)
        outs.append((x.readback_hdr_f32().astype(np.float64), x.readback_depth()))
    (h, depth) = outs[0]
    if len(outs) > 1:
        assert np.array_equal(depth.view(np.uint32), outs[1][1].view(np.uint32)), "depth differs from the oracle"
    bnd = sky.bounds()[0]
    with np.errstate(invalid="ignore"):
        lo, hi = f16(sky.value - bnd), f16(sky.value + bnd)

    def blend(dst):
        a = f32(src[3])
        rgb = (src[:3] * a).astype(f32) + (dst[..., :3].astype(f32) * f32(1.0 - a)).astype(f32)
        return np.concatenate([f16(rgb), np.broadcast_to(f16(f32(a + f32(1.0 - a))), dst.shape[:-1] + (1,))], axis=-1)

    blo, bhi = blend(lo), blend(hi)
    full = (depth > 0) & ok_sky
    assert np.count_nonzero(full) > 300 and np.count_nonzero(depth == 0) > 300
    with np.errstate(invalid="ignore"):
        inside = (blo <= h) & (h <= bhi)
    bad = full & ~inside.all(-1)
    assert not bad.any(), f"{samples}x: {np.count_nonzero(bad)} blended pixels are not R8 over the f16 sky, first at {np.argwhere(bad)[0]}"
    if samples == 4:
        part = (depth == 0) & ok_sky & ~np.all((lo <= h) & (h <= hi), axis=-1)
        lo_all, hi_all = np.minimum(lo, blo), np.maximum(hi, bhi)
        slack = 4 * U * np.abs(np.where(np.isfinite(hi_all), hi_all, 0.0))
        with np.errstate(invalid="ignore"):
            between = ((lo_all - slack <= h) & (h <= hi_all + slack)).all(-1)
        assert np.count_nonzero(part) > 10 and not (part & ~between).any(), "a partly covered 4x pixel is not between sky and layer"


# ------------------------------------------------------------------ the Python mirror's face check
def test_set_skybox_rejects_faces_that_are_not_one_square_size():
    """wgpu rejects a cube texture whose faces are not equal squares; so does Renderer.set_skybox, which would otherwise hand the
    library one width for faces of several shapes."""
    ok = [np.zeros((4, 4, 4), dtype=np.uint8)] * 6
    Renderer().set_skybox(ok)
    Renderer().set_skybox([np.zeros((4, 4, 4), dtype=np.float32)] * 6)
    Renderer().set_skybox(None)
    bad = {
        "non-square": [np.zeros((4, 8, 4), dtype=np.uint8)] * 6,
        "sizes differ": ok[:5] + [np.zeros((8, 8, 4), dtype=np.uint8)],
        "dtypes differ": ok[:5] + [np.zeros((4, 4, 4), dtype=np.float32)],
        "five faces": ok[:5],
        "three channels": [np.zeros((4, 4, 3), dtype=np.uint8)] * 6,
        "float64": [np.zeros((4, 4, 4), dtype=np.float64)] * 6,
        "empty": [np.zeros((0, 0, 4), dtype=np.uint8)] * 6,
    }
    for what, faces in bad.items():
        with pytest.raises(ValueError, match="set_skybox"):
            Renderer().set_skybox(faces)


# ------------------------------------------------------------------ g. graph-submitted frames
@pytest.mark.gpu
def test_sky_in_graph_frames():
    """Two frames submitted as one CUDA graph each, the camera turned between them: the second frame's sky is the reference's for the
    new camera and the same bits as a frame rendered without the graph."""
    from rend3_b200.backend import load_cuda_backend

    v = sk.SkyView(sk.random_faces(64, "rgba8_srgb", 31), srgb=True, view=sk.random_rotation(32), projection=("perspective", 70.0, 0.1), resolution=(80, 60))
    turned = sk.random_rotation(33)
    g, plain = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    try:
        r = sk.runner(g, v)
        sk.draw(r, v.resolution, frame_graph=True)
        first = g.readback_hdr_f32().copy()
        sref.compare(first, sk.reference(r, v.resolution), "graph frame 0")
        r.renderer.set_camera_data(sk.Camera(v.projection, turned))
        sk.draw(r, v.resolution, frame_graph=True, upload=False)
        second = g.readback_hdr_f32()
        sky = sk.reference(r, v.resolution)
        sref.compare(second, sky, "graph frame 1")
        assert not np.array_equal(first, second), "the turned camera must change the sky"
        _, _ = sk.render(plain, dataclasses.replace(v, view=turned))
        assert np.array_equal(second.view(np.uint32), plain.readback_hdr_f32().view(np.uint32)), "graph and plain frames differ"
    finally:
        g.close()
        plain.close()
