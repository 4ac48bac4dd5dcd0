"""Float64 restatement of skybox.wgsl's fs_main (rend3-routine/shaders/src/skybox.wgsl:24-36) with the cube sampling of rule R10
(DESIGN.md), written from the Vulkan cube-map face table and rule R9's trilinear filter, not from the oracle or the kernels.

Inputs are what the kernels read: the frame uniform's `inv_origin_view_proj` as its sixteen f32 words (column-major, word 4 c + r),
the target size, the sky's `r3_texture_desc` and the raw texel blob.  Mip generation is not part of it: the levels are read from the
blob as stored.

Per pixel, in float64:
  * the direction at the pixel centre: NDC (cx, cy) = ((px + 0.5) / (W / 2) - 1, 1 - (py + 0.5) / (H / 2)), then
    M (cx, cy, 1, 1), divided by w, normalised;
  * the face by the major axis, exact ties X over Y over Z;
  * (s, t) = ((sc / |rc| + 1) / 2, (tc / |rc| + 1) / 2) with (sc, tc, rc) from the Vulkan table (FACES below);
  * forward differences of (s, t) at (px + 1.5, py + 0.5) and (px + 0.5, py + 1.5), both projected onto the centre's face;
  * rho = the larger Euclidean length of the derivatives scaled by the level-0 width, lambda = log2(rho) exactly;
  * level 0 when lambda <= 0, else trilinear between floor(l) and floor(l) + 1 with l = min(lambda, mip_count - 1); bilinear at
    (s w - 0.5, t w - 0.5) with texels clamped to the face; RGBA8 sRGB decoded per texel by the IEC 61966-2-1 curve; alpha 1.

Alongside the value it returns what the error bound needs (see `Sky.bound_of`): the f32 error of the direction and of (s, t), the
error of lambda, the texel range of every footprint the f32 path could fetch, a flag for pixels whose face the f32 path may pick
differently (with the value of the other candidate face), and a flag for pixels whose fetched texels are not fixed by the f32
error (there a non-finite texel may or may not be read)."""
from dataclasses import dataclass

import numpy as np

from rend3_b200.layouts import TEXFMT_RGBA8_UNORM_SRGB, TEXFMT_RGBA32_FLOAT

U = 2.0 ** -24                     # unit roundoff of f32
LOG2_R9 = 4e-7                     # rule R9's log2: |error| < 4e-7 (tests/test_host_cpu.py pins it)

# Vulkan specification, "Cube Map Face Selection and Transformations": layer, major axis, sign, and the vectors whose dot product
# with the direction gives sc and tc
FACES = [
    (0, +1, (0, 0, -1), (0, -1, 0)),   # +X: sc = -rz, tc = -ry
    (0, -1, (0, 0, +1), (0, -1, 0)),   # -X: sc = +rz, tc = -ry
    (1, +1, (+1, 0, 0), (0, 0, +1)),   # +Y: sc = +rx, tc = +rz
    (1, -1, (+1, 0, 0), (0, 0, -1)),   # -Y: sc = +rx, tc = -rz
    (2, +1, (+1, 0, 0), (0, -1, 0)),   # +Z: sc = +rx, tc = -ry
    (2, -1, (-1, 0, 0), (0, -1, 0)),   # -Z: sc = -rx, tc = -ry
]


def srgb_decode(e):
    return np.where(e > 0.04045, ((e + 0.055) / 1.055) ** 2.4, e / 12.92)


def face_levels(desc, blob):
    """levels[face][level] = (w, w, 4) float64 texels of the six faces, read from the blob as the descriptor places them."""
    w0, n, fmt, off = int(desc["width"]), int(desc["mip_count"]), int(desc["format"]), int(desc["byte_offset"])
    bpp = 16 if fmt == TEXFMT_RGBA32_FLOAT else 4
    blob = np.asarray(blob).view(np.uint8).reshape(-1)
    out = []
    for _ in range(6):
        levels = []
        for l in range(n):
            w = max(w0 >> l, 1)
            raw = blob[off:off + w * w * bpp]
            off += w * w * bpp
            if fmt == TEXFMT_RGBA32_FLOAT:
                t = raw.view(np.float32).reshape(w, w, 4).astype(np.float64)
            else:
                t = raw.reshape(w, w, 4).astype(np.float64) / 255.0
                if fmt == TEXFMT_RGBA8_UNORM_SRGB:
                    t[..., :3] = srgb_decode(t[..., :3])
            levels.append(t)
        out.append(levels)
    return out


def directions(m, width, height, fx, fy):
    """Unit directions at the framebuffer points (fx, fy) and a bound on the f32 path's absolute error per component.

    The f32 path computes cx, cy with one division and one subtraction (|error| <= 4u), the product M (cx, cy, 1, 1) as four
    products summed in order (|error| <= 4u sum_c |M_cr| |clip_c| plus |M_0r| + |M_1r| times the error of cx, cy), the division
    by w (first order: (E_i + |v_i| E_w) / |w| + u |v_i|) and the normalisation (a relative 4u on each component plus the part of
    the error of v across the direction, |dv| / |v|).  The sum is doubled, so that the bound does not rest on counting every
    rounding exactly; second-order terms are far smaller."""
    cx, cy = fx / (width * 0.5) - 1.0, 1.0 - fy / (height * 0.5)
    clip = np.stack([cx, cy, np.ones_like(cx), np.ones_like(cx)], axis=-1)
    wu = clip @ m                                               # m[c, r]: wu_r = sum_c m[c, r] clip_c
    e = 4 * U * (np.abs(clip) @ np.abs(m)) + 4 * U * (np.abs(m[0]) + np.abs(m[1]))
    v = wu[..., :3] / wu[..., 3:]
    dv = (e[..., :3] + np.abs(v) * e[..., 3:]) / np.abs(wu[..., 3:]) + U * np.abs(v)
    n = np.linalg.norm(v, axis=-1, keepdims=True)
    err = 2.0 * (np.linalg.norm(dv, axis=-1) / n[..., 0] + 4 * U)
    return v / n, err


def project(d, err, face):
    """(s, t) of direction(s) d on `face` (array of face indices) and the bound on their f32 error: q = sc / |rc| is off by
    (|dsc| + |q| |drc|) / |rc| + u |q|, s = (q + 1) / 2 by half that plus the rounding of q + 1."""
    axis = np.array([f[0] for f in FACES])[face]
    svec = np.array([f[2] for f in FACES], dtype=np.float64)[face]
    tvec = np.array([f[3] for f in FACES], dtype=np.float64)[face]
    ma = np.abs(np.take_along_axis(d, axis[..., None], axis=-1)[..., 0])
    qs, qt = (d * svec).sum(-1) / ma, (d * tvec).sum(-1) / ma
    es = 0.5 * (err * (1 + np.abs(qs)) / ma + U * (np.abs(qs) + np.abs(qs + 1)))
    et = 0.5 * (err * (1 + np.abs(qt)) / ma + U * (np.abs(qt) + np.abs(qt + 1)))
    return 0.5 * (qs + 1.0), 0.5 * (qt + 1.0), np.maximum(es, et)


def face_of(d):
    """Rule R10's face: the major axis, exact ties X over Y over Z; and the face of the runner-up axis."""
    a = np.abs(d)
    axis = np.where((a[..., 0] >= a[..., 1]) & (a[..., 0] >= a[..., 2]), 0, np.where(a[..., 1] >= a[..., 2], 1, 2))
    masked = a.copy()
    np.put_along_axis(masked, axis[..., None], -1.0, axis=-1)
    second = masked.argmax(-1)
    sign_face = lambda ax: 2 * ax + (np.take_along_axis(d, ax[..., None], axis=-1)[..., 0] <= 0)
    gap = np.take_along_axis(a, axis[..., None], -1)[..., 0] - np.take_along_axis(a, second[..., None], -1)[..., 0]
    return sign_face(axis), sign_face(second), gap


def bilinear(tex, s, t):
    """Bilinear at (s w - 0.5, t w - 0.5), texels clamped to the face, in IEEE arithmetic (an infinite texel with weight 0 gives NaN
    as it does in f32)."""
    w = tex.shape[0]
    x, y = s * w - 0.5, t * w - 0.5
    x0, y0 = np.floor(x), np.floor(y)
    fx, fy = (x - x0)[..., None], (y - y0)[..., None]
    ix0, iy0 = np.clip(x0, 0, w - 1).astype(int), np.clip(y0, 0, w - 1).astype(int)
    ix1, iy1 = np.clip(x0 + 1, 0, w - 1).astype(int), np.clip(y0 + 1, 0, w - 1).astype(int)
    return (tex[iy0, ix0] * (1 - fx) + tex[iy0, ix1] * fx) * (1 - fy) + (tex[iy1, ix0] * (1 - fx) + tex[iy1, ix1] * fx) * fy


def footprint_range(tex, s, t, dxy):
    """Per channel (min, max, max |texel|, any non-finite texel) over every 2 x 2 footprint the bilinear fetch can take when its
    coordinates move by up to dxy texels (non-finite texels left out of the first three), and whether that is more than one
    footprint."""
    w = tex.shape[0]
    x, y = s * w - 0.5, t * w - 0.5
    xa, xb, ya, yb = np.floor(x - dxy), np.floor(x + dxy) + 1, np.floor(y - dxy), np.floor(y + dxy) + 1
    cols = np.clip(np.minimum(xa[..., None] + np.arange(3), xb[..., None]), 0, w - 1).astype(int)
    rows = np.clip(np.minimum(ya[..., None] + np.arange(3), yb[..., None]), 0, w - 1).astype(int)
    block = tex[rows[..., :, None], cols[..., None, :]]          # (..., 3, 3, 4)
    fin = np.isfinite(block).all(axis=(-3, -2))
    b = np.where(np.isfinite(block), block, 0.0)
    big = np.abs(b).max(axis=(-3, -2))
    moved = (xb - xa > 2) | (yb - ya > 2)
    return b.min(axis=(-3, -2)), b.max(axis=(-3, -2)), big, ~fin, moved


@dataclass
class Sampled:
    value: np.ndarray       # (..., 4)
    lam: np.ndarray         # lambda (exact log2 of rho)
    eps_st: np.ndarray      # f32 error bound of (s, t) and of the projected neighbours
    eps_lam: np.ndarray
    rng: np.ndarray         # (..., 4) texel range over every footprint the f32 path can fetch, on every level it can read
    big: np.ndarray         # (..., 4) max |texel| there
    nonfinite: np.ndarray   # (..., 4) a non-finite texel among them
    moved: np.ndarray       # the fetched texels are not fixed by the f32 error
    w_level: np.ndarray     # width of the finest level the sample can read


def sample_face(levels, face, d0, e0, dx, ex, dy, ey):
    """textureSample(cube, direction) on `face` (one index per pixel) with rule R10's derivatives."""
    s, t, es0 = project(d0, e0, face)
    sx, tx, esx = project(dx, ex, face)
    sy, ty, esy = project(dy, ey, face)
    w0 = levels[0][0].shape[0]
    last = len(levels[0]) - 1
    jx, jy = np.hypot(sx - s, tx - t) * w0, np.hypot(sy - s, ty - t) * w0
    rho = np.maximum(jx, jy)
    with np.errstate(divide="ignore"):
        lam = np.log2(rho)
    # the f32 derivative is off by the errors of both points (plus its own rounding), so rho by sqrt(2) w0 times their sum
    drho = np.sqrt(2.0) * w0 * (es0 + np.maximum(esx, esy)) + 4 * U * rho
    r = drho / np.maximum(rho, 1e-300)
    with np.errstate(divide="ignore", invalid="ignore"):
        eps_lam = np.where(r < 1, -np.log2(np.maximum(1 - r, 1e-300)), np.inf) + LOG2_R9 + 2 * U * np.abs(lam)
    eps_st = np.maximum(es0, np.maximum(esx, esy))
    shape = s.shape
    value = np.zeros(shape + (4,))
    tmin, tmax, big = np.full(shape + (4,), np.inf), np.full(shape + (4,), -np.inf), np.zeros(shape + (4,))
    nonfinite = np.zeros(shape + (4,), dtype=bool)
    moved = np.zeros(shape, dtype=bool)
    w_level = np.zeros(shape)
    l_nom = np.minimum(lam, last)
    lo_nom = np.where(lam > 0, np.floor(l_nom), 0).astype(int)
    fr = np.where(lam > 0, l_nom - np.floor(l_nom), 0.0)
    # levels any lambda within eps_lam can read
    lam_lo, lam_hi = lam - eps_lam, lam + eps_lam
    lv_lo = np.where(lam_lo > 0, np.floor(np.minimum(lam_lo, last)), 0).astype(int)
    lv_hi = np.where(lam_hi > 0, np.minimum(np.floor(np.minimum(lam_hi, last)) + 1, last), 0).astype(int)
    hi_nom = np.where((fr != 0) & (lo_nom < last), lo_nom + 1, lo_nom)
    moved |= (lv_lo != lo_nom) | (lv_hi != hi_nom)
    with np.errstate(invalid="ignore", over="ignore"):
        for f in range(6):
            for l in range(last + 1):
                tex = levels[f][l]
                here = face == f
                if not here.any():
                    continue
                a = bilinear(tex, s, t)
                sel = here & (lo_nom == l)
                if sel.any():
                    b = bilinear(levels[f][min(l + 1, last)], s, t)
                    g = fr[..., None]
                    tri = np.where((g == 0) | (l >= last), a, a * (1 - g) + b * g)
                    value[sel] = tri[sel]
                used = here & (lv_lo <= l) & (l <= lv_hi)
                if used.any():
                    wl = tex.shape[0]
                    lo, hi, bg, nf, mv = footprint_range(tex, s, t, wl * (eps_st + 4 * U))
                    tmin[used] = np.minimum(tmin[used], lo[used])
                    tmax[used] = np.maximum(tmax[used], hi[used])
                    big[used] = np.maximum(big[used], bg[used])
                    nonfinite[used] |= nf[used]
                    moved[used] |= mv[used]
                    w_level[used] = np.maximum(w_level[used], wl)
    value[..., 3] = 1.0
    nonfinite[..., 3] = False
    return Sampled(value, lam, eps_st, eps_lam, tmax - tmin, big, nonfinite, moved, w_level)


@dataclass
class Sky:
    """The reference sky of one frame, (H, W) per pixel."""
    face: np.ndarray        # rule R10's face
    other: np.ndarray       # the runner-up axis's face
    flagged: np.ndarray     # the f32 path may pick `other` (the two largest |components| closer than their f32 errors)
    exact_tie: np.ndarray   # the two largest |components| are equal in float64 (constructed ties: the rule decides)
    seam: np.ndarray        # the right or lower neighbour's direction lies on another face
    main: Sampled
    alt: Sampled
    last: int

    @property
    def value(self):
        return self.main.value

    @staticmethod
    def bound_of(smp: Sampled):
        """|x - ref| <= 1e-4 max(1, |ref|) + R (w_level (eps_st + 4u) + eps_lam) + 8u A.

        Away from face ties the sample is a continuous function of (s, t) and lambda: bilinear weights are continuous in the
        coordinates (a texel enters the footprint with weight 0), the trilinear blend is continuous at integer lambda, at lambda <= 0
        and at the clamp to the last level.  Its slope along a coordinate measured in texels is at most the footprint's texel range R,
        and along lambda at most the range between the two levels' footprints, also within R (R is taken over every footprint the f32
        path can fetch, on every level it can read).  A coordinate in texels is off by w_level (eps_st + 4u): (s, t) by eps_st, the
        product s w and the subtraction of 0.5 by 4u w.  Lambda is off by eps_lam: rule R9's log2 (< 4e-7), the rounding of rho and the
        error of the forward differences, which the f32 path takes between two points that carry eps_st each.  8u A (A = max |texel|
        of the footprint) covers the roundings of the f32 lerps, and 1e-4 max(1, |ref|) the per-texel decode (sRGB's powf, 1/255)."""
        return 1e-4 * np.maximum(1.0, np.abs(smp.value)) + smp.rng * (smp.w_level * (smp.eps_st + 4 * U) + smp.eps_lam)[..., None] \
            + 8 * U * smp.big

    def bounds(self):
        return self.bound_of(self.main), self.bound_of(self.alt)


def reference_sky(inv_origin_view_proj, width, height, desc, blob):
    m = np.asarray(inv_origin_view_proj, dtype=np.float32).astype(np.float64).reshape(4, 4)
    levels = face_levels(desc, blob)
    py, px = np.mgrid[0:height, 0:width].astype(np.float64)
    d0, e0 = directions(m, width, height, px + 0.5, py + 0.5)
    dx, ex = directions(m, width, height, px + 1.5, py + 0.5)
    dy, ey = directions(m, width, height, px + 0.5, py + 1.5)
    face, other, gap = face_of(d0)
    exact_tie = gap == 0
    flagged = (gap <= 2 * e0) & ~exact_tie
    seam = (face_of(dx)[0] != face) | (face_of(dy)[0] != face)
    main = sample_face(levels, face, d0, e0, dx, ex, dy, ey)
    alt = sample_face(levels, other, d0, e0, dx, ex, dy, ey)
    return Sky(face, other, flagged, exact_tie, seam, main, alt, len(levels[0]) - 1)


@dataclass
class Comparison:
    worst_ratio: float      # max |x - ref| / bound over the finite values compared
    n_flagged: int          # pixels where either candidate face was accepted
    n_skipped: int          # pixels with a non-finite texel among footprints the f32 error leaves open (NaN / inf not decided)


def compare(got, sky: Sky, what="", mask=None):
    """Assert `got` (H, W, 4) is the reference sky within the bound; a flagged pixel may match either candidate face.  Non-finite
    values: where the footprint holds a non-finite texel and the fetched texels are fixed, `got` is NaN exactly where the reference
    is NaN and equals it where it is infinite.  `mask` restricts the comparison to the pixels the sky covers."""
    got = np.asarray(got, dtype=np.float64)
    ratios = []
    ok_pixels = []
    skipped = np.zeros(sky.face.shape, dtype=bool)
    for smp, b in zip((sky.main, sky.alt), sky.bounds()):
        ref = smp.value
        nf = smp.nonfinite
        open_ = nf.any(-1) & smp.moved
        with np.errstate(invalid="ignore"):
            err = np.abs(got - ref)
            fin_ok = np.where(nf, True, err <= b)
            nan_ok = np.where(nf, (np.isnan(got) == np.isnan(ref)) & (np.isnan(ref) | np.isfinite(ref) & (err <= b) | (got == ref)), True)
        ok = (fin_ok & nan_ok).all(-1) | open_
        ok_pixels.append(ok)
        skipped |= open_
        with np.errstate(invalid="ignore", divide="ignore"):
            ratios.append(np.where(~nf & np.isfinite(b), err / b, 0.0))
    ok = ok_pixels[0] | (sky.flagged & ok_pixels[1])
    if mask is not None:
        ok |= ~mask
    bad = ~ok
    assert not bad.any(), f"{what}: {np.count_nonzero(bad)} pixels outside the reference's bound; first at {np.argwhere(bad)[0]}: " \
                          f"got {got[tuple(np.argwhere(bad)[0])]}, want {sky.value[tuple(np.argwhere(bad)[0])]} " \
                          f"(face {sky.face[tuple(np.argwhere(bad)[0])]}, bound {sky.bounds()[0][tuple(np.argwhere(bad)[0])]})"
    main_ok = ok_pixels[0] & ~skipped
    worst = float(np.max(ratios[0][main_ok], initial=0.0))
    return Comparison(worst, int(np.count_nonzero(sky.flagged)), int(np.count_nonzero(skipped)))
