"""textureSampleGrad on the 2D texture table and get_pixel_data_inner, restated in float64 numpy from opaque.wgsl:203-424,
depth.wgsl:101-127, the Vulkan filtering rules (level of detail, bilinear footprint, Repeat addressing) and the text of rule R9
(DESIGN.md §2).  It is not derived from rend3_b200/csrc/r3_texture.cuh or the oracle.

Inputs are what the kernels read: a `r3_texture_desc` row of the table, the raw texel blob (levels read as stored: mip generation
is not restated) and the material record as the kernels receive it.  Texels decode through the float64 decoders of the package
(`bc.decode` for the block formats, `texformats.unpack` for formats 17 - 30) and unorm / 255 with the IEC 61966-2-1 curve for the
five common formats; missing channels read (0, 0, 1).

Per sample, in float64:
  * rho = the larger Euclidean length of (du/dx w0, dv/dx h0) and (du/dy w0, dv/dy h0), lambda = log2(rho) exactly;
  * linear sampler: level 0 when lambda <= 0, else trilinear between floor(l) and floor(l) + 1 with l = min(lambda, mip_count - 1),
    one level where the fraction is 0 or the level is the last;
  * nearest sampler: level floor(lambda + 0.5) clamped to the last (0 when lambda <= 0), texel floor(u w);
  * bilinear footprint at (u w - 0.5, v h - 0.5) with Repeat: texel i of a row of n is i mod n, also for negative i.

Alongside the value it returns what an error bound needs, as tests/skybox_reference.py does for the sky: the error of lambda
(rule R9's log2 plus the error of the derivatives), the texel range over every footprint the f32 coordinates can fetch on every
level they can read, a flag where the nearest sampler's level is not fixed by the f32 error (lambda within its error of k + 0.5,
with the value at the other candidate level), and a flag where a non-finite texel may or may not be fetched."""
from dataclasses import dataclass

import numpy as np

from rend3_b200 import bc, texformats
from rend3_b200.layouts import (MAT_AOMR_BW_SPLIT, MAT_AOMR_COMBINED, MAT_AOMR_SWIZZLED_SPLIT, MAT_ALBEDO_ACTIVE, MAT_ALBEDO_BLEND,
                                MAT_ALBEDO_VERTEX_SRGB, MAT_CC_GLTF_COMBINED, MAT_CC_GLTF_SPLIT, MAT_NEAREST,
                                MAT_UNLIT, MATERIAL_DTYPE, TEX_ALBEDO, TEX_AMBIENT_OCCLUSION, TEX_CLEAR_COAT, TEX_CLEAR_COAT_ROUGHNESS,
                                TEX_EMISSIVE, TEX_METALLIC, TEX_NORMAL, TEX_REFLECTANCE, TEX_ROUGHNESS, TEXFMT_R8_UNORM, TEXFMT_RG8_UNORM,
                                TEXFMT_RGBA32_FLOAT, TEXFMT_RGBA8_UNORM, TEXFMT_RGBA8_UNORM_SRGB, texfmt_element_bytes, texfmt_level_shape)
from skybox_reference import LOG2_R9, U, srgb_decode
import vertex_reference as vref

_BLOCK = {}
for _name, (_plain, _srgb, _) in bc.BLOCK_FORMATS.items():
    _BLOCK[_plain] = (_name, False)
    if _srgb is not None:
        _BLOCK[_srgb] = (_name, True)
_WIDE = {fmt: name for name, (fmt, _) in texformats.STORAGE.items()}


# ------------------------------------------------------------------ texels
def texture_levels(desc, blob):
    """levels[l] = (h_l, w_l, 4) float64 texels of one table entry, read from the blob where the descriptor places them: level l is
    max(w >> l, 1) x max(h >> l, 1) and follows level l - 1 directly."""
    w0, h0, n, fmt, off = (int(desc[k]) for k in ("width", "height", "mip_count", "format", "byte_offset"))
    blob = np.asarray(blob).view(np.uint8).reshape(-1)
    out = []
    for l in range(n):
        w, h, cols, rows = texfmt_level_shape(fmt, w0, h0, l)
        nbytes = cols * rows * texfmt_element_bytes(fmt)
        raw = blob[off:off + nbytes]
        off += nbytes
        if fmt in _BLOCK:
            name, srgb = _BLOCK[fmt]
            t = bc.decode(name, raw, w, h, srgb=srgb)
        elif fmt in _WIDE:
            t = texformats.unpack(_WIDE[fmt], raw, w, h)
        elif fmt == TEXFMT_RGBA32_FLOAT:
            t = raw.view(np.float32).reshape(h, w, 4).astype(np.float64)
        else:
            c = {TEXFMT_R8_UNORM: 1, TEXFMT_RG8_UNORM: 2}.get(fmt, 4)
            t = np.zeros((h, w, 4))
            t[..., 3] = 1.0
            t[..., :c] = raw.reshape(h, w, c).astype(np.float64) / 255.0
            if fmt == TEXFMT_RGBA8_UNORM_SRGB:
                t[..., :3] = srgb_decode(t[..., :3])
            assert fmt in (TEXFMT_RGBA8_UNORM, TEXFMT_RGBA8_UNORM_SRGB, TEXFMT_R8_UNORM, TEXFMT_RG8_UNORM), fmt
        out.append(t)
    return out


class Table:
    """The texture table: descriptors and blob; levels decoded once per entry."""

    def __init__(self, descs, blob):
        self.descs, self.blob, self._levels = descs, blob, {}

    def levels(self, slot_value):
        """The levels of a material slot's texture (slot value = table index + 1), None where the slot is 0 or past the table."""
        if slot_value == 0 or slot_value > len(self.descs):
            return None
        if slot_value not in self._levels:
            self._levels[slot_value] = texture_levels(self.descs[slot_value - 1], self.blob)
        return self._levels[slot_value]


def bilinear(tex, u, v):
    """Bilinear at (u w - 0.5, v h - 0.5) with Repeat, in IEEE arithmetic."""
    h, w = tex.shape[:2]
    x, y = u * w - 0.5, v * h - 0.5
    x0, y0 = np.floor(x), np.floor(y)
    fx, fy = (x - x0)[..., None], (y - y0)[..., None]
    ix0, iy0 = np.mod(x0, w).astype(np.int64), np.mod(y0, h).astype(np.int64)
    ix1, iy1 = np.mod(x0 + 1, w).astype(np.int64), np.mod(y0 + 1, h).astype(np.int64)
    return (tex[iy0, ix0] * (1 - fx) + tex[iy0, ix1] * fx) * (1 - fy) + (tex[iy1, ix0] * (1 - fx) + tex[iy1, ix1] * fx) * fy


def nearest(tex, u, v):
    h, w = tex.shape[:2]
    return tex[np.mod(np.floor(v * h), h).astype(np.int64), np.mod(np.floor(u * w), w).astype(np.int64)]


def footprint_range(tex, u, v, dxy, linear):
    """Per channel (min, max, max |texel|, any non-finite texel) over every footprint the fetch can take when its coordinates move by
    up to dxy texels (non-finite texels left out of the first three), and whether that is more than one footprint.  A reach wider than
    four texels takes the whole level."""
    h, w = tex.shape[:2]
    x, y = (u * w - 0.5, v * h - 0.5) if linear else (u * w, v * h)
    xa, ya = np.floor(x - dxy), np.floor(y - dxy)
    xb, yb = np.floor(x + dxy) + linear, np.floor(y + dxy) + linear
    wide = (xb - xa >= 4) | (yb - ya >= 4)
    cols = np.mod(np.minimum(xa[..., None] + np.arange(4), xb[..., None]), w).astype(np.int64)
    rows = np.mod(np.minimum(ya[..., None] + np.arange(4), yb[..., None]), h).astype(np.int64)
    block = tex[rows[..., :, None], cols[..., None, :]]            # (..., 4, 4, 4)
    fin = np.isfinite(block)
    b = np.where(fin, block, 0.0)
    lo, hi, big, nf = b.min(axis=(-3, -2)), b.max(axis=(-3, -2)), np.abs(b).max(axis=(-3, -2)), ~fin.all(axis=(-3, -2))
    if wide.any():
        tf = np.isfinite(tex)
        tb = np.where(tf, tex, 0.0)
        lo[wide], hi[wide] = tb.min(axis=(0, 1)), tb.max(axis=(0, 1))
        big[wide], nf[wide] = np.abs(tb).max(axis=(0, 1)), ~tf.all(axis=(0, 1))
    moved = (xb - xa > linear) | (yb - ya > linear)
    return lo, hi, big, nf, moved


@dataclass
class Sampled:
    value: np.ndarray       # (N, 4)
    lam: np.ndarray         # lambda, exact log2 of rho
    eps_lam: np.ndarray     # its f32 error: rule R9's log2, the rounding of rho, the error of the derivatives
    level: np.ndarray       # the level read (the lower one of a trilinear pair)
    fr: np.ndarray          # the trilinear fraction (0 for the nearest sampler)
    tie: np.ndarray         # nearest sampler: lambda within eps_lam of k + 0.5 (either level may be read)
    alt: np.ndarray         # (N, 4) the value at the other candidate level where `tie`
    rng: np.ndarray         # (N, 4) texel range over every footprint the f32 path can fetch, on every level it can read
    big: np.ndarray         # (N, 4) max |texel| there
    nonfinite: np.ndarray   # (N, 4) a non-finite texel among them
    moved: np.ndarray       # the fetched texels are not fixed by the f32 error
    texels: np.ndarray      # (N,) coordinate error in texels of the finest level read
    linear: bool

    def bound(self):
        """|x - value| <= 1e-4 max(1, |value|) + R (texels + eps_lam) + 8u A (linear sampler), 1e-4 max(1, |value|) + R [moved]
        (nearest).  Linear: the sample is continuous in the coordinates and in lambda (a texel enters the footprint with weight 0; the
        trilinear blend is continuous at integer lambda, at lambda <= 0 and at the last level), with slope at most the texel range R
        along a coordinate measured in texels and along lambda.  Nearest: the value is one texel; where the coordinate error can
        move the texel, any texel of the range.  8u A covers the f32 lerps, 1e-4 the per-texel decode (sRGB's powf, the divisions)."""
        base = 1e-4 * np.maximum(1.0, np.abs(self.value))
        if self.linear:
            return base + self.rng * (self.texels + self.eps_lam)[..., None] + 8 * U * self.big
        return base + np.where(self.moved[..., None], self.rng, 0.0)


def sample_grad(levels, linear, u, v, dudx, dvdx, dudy, dvdy, eps_c, eps_d):
    """textureSampleGrad(levels, sampler, (u, v), (dudx, dvdx), (dudy, dvdy)) for N fragments.  eps_c bounds the f32 error of the
    coordinates, eps_d that of the derivatives (both in texture-coordinate units)."""
    n = np.shape(u)[0]
    h0, w0 = levels[0].shape[:2]
    last = len(levels) - 1
    rho = np.maximum(np.hypot(dudx * w0, dvdx * h0), np.hypot(dudy * w0, dvdy * h0))
    with np.errstate(divide="ignore", invalid="ignore"):
        lam = np.log2(rho)
        drho = np.sqrt(2.0) * max(w0, h0) * eps_d + 4 * U * rho
        r = drho / np.maximum(rho, 1e-300)
        eps_lam = np.where(r < 1, -np.log2(np.maximum(1 - r, 1e-300)), np.inf) + LOG2_R9 + 2 * U * np.abs(np.nan_to_num(lam, neginf=0.0))
    pos = lam > 0
    tie = np.zeros(n, dtype=bool)
    fr = np.zeros(n)
    if linear:
        l = np.minimum(lam, last)
        level = np.where(pos, np.floor(l), 0).astype(np.int64)
        fr = np.where(pos, l - np.floor(l), 0.0)
        hi_level = np.where((fr != 0) & (level < last), level + 1, level)
        lam_lo, lam_hi = lam - eps_lam, lam + eps_lam
        lv_lo = np.where(lam_lo > 0, np.floor(np.minimum(lam_lo, last)), 0).astype(np.int64)
        lv_hi = np.where(lam_hi > 0, np.minimum(np.floor(np.minimum(lam_hi, last)) + 1, last), 0).astype(np.int64)
        other = level
    else:
        pick = lambda x: np.where(x > 0, np.minimum(np.floor(x + 0.5), last), 0).astype(np.int64)
        level = hi_level = pick(lam)
        lv_lo, lv_hi = pick(lam - eps_lam), pick(lam + eps_lam)
        tie = lv_lo != lv_hi
        other = np.where(lv_lo != level, lv_lo, lv_hi)
    moved = (lv_lo != level) | (lv_hi != hi_level)
    value, alt = np.zeros((n, 4)), np.zeros((n, 4))
    tmin, tmax, big = np.full((n, 4), np.inf), np.full((n, 4), -np.inf), np.zeros((n, 4))
    nonfinite = np.zeros((n, 4), dtype=bool)
    texels = np.zeros(n)
    fetch = bilinear if linear else nearest
    with np.errstate(invalid="ignore", over="ignore"):
        for lv in range(last + 1):
            tex = levels[lv]
            sel = level == lv
            if sel.any():
                a = fetch(tex, u[sel], v[sel])
                if linear:
                    b = bilinear(levels[min(lv + 1, last)], u[sel], v[sel])
                    g = fr[sel][:, None]
                    a = np.where((g == 0) | (lv >= last), a, a * (1 - g) + b * g)
                value[sel] = a
            osel = tie & (other == lv)
            if osel.any():
                alt[osel] = fetch(tex, u[osel], v[osel])
            used = (lv_lo <= lv) & (lv <= lv_hi)
            if used.any():
                hl, wl = tex.shape[:2]
                # the coordinate error in texels, plus the roundings of u w and of the subtraction of 0.5
                dt = max(wl, hl) * eps_c[used] + 2 * U * (max(wl, hl) * np.maximum(np.abs(u[used]), np.abs(v[used])) + 1)
                lo, hi, bg, nf, mv = footprint_range(tex, u[used], v[used], dt, int(linear))
                tmin[used], tmax[used] = np.minimum(tmin[used], lo), np.maximum(tmax[used], hi)
                big[used] = np.maximum(big[used], bg)
                nonfinite[used] |= nf
                moved[used] |= mv
                texels[used] = np.maximum(texels[used], dt)
    return Sampled(value, lam, eps_lam, level, fr, tie, alt, tmax - tmin, big, nonfinite, moved, texels, linear)


def sample_slot(table: Table, slot_value, linear, c):
    """Sampled of one material slot at TexCoords `c` (see `coords`); a slot past the table gives zeros with a zero bound."""
    levels = table.levels(slot_value)
    n = len(c.u)
    if levels is None:
        z = np.zeros((n, 4))
        return Sampled(z, np.zeros(n), np.zeros(n), np.zeros(n, np.int64), np.zeros(n), np.zeros(n, bool), z, z, z, np.zeros((n, 4), bool),
                       np.zeros(n, bool), np.zeros(n), linear)
    return sample_grad(levels, linear, c.u, c.v, c.dudx, c.dvdx, c.dudy, c.dvdy, c.eps_c, c.eps_d)


# ------------------------------------------------------------------ texture coordinates (rule R6 at three pixel centres, rule R9)
@dataclass
class TexCoords:
    u: np.ndarray
    v: np.ndarray
    dudx: np.ndarray
    dvdx: np.ndarray
    dudy: np.ndarray
    dvdy: np.ndarray
    eps_c: np.ndarray       # f32 error bound of (u, v)
    eps_d: np.ndarray       # f32 error bound of the forward differences


def uv_transform(rec):
    """uv_transform0 as float64 t[column][row] (3, 3)."""
    return np.asarray(rec["uv_transform0"], dtype=np.float32).astype(np.float64)[:, :3]


def coords(xyw, uv_tri, fx, fy, width, height, t=None, depth_pass=False):
    """TexCoords of fragments of one triangle whose unclipped clip xyw are `xyw` (3, 3) and whose uv0 are `uv_tri` (3, 2), shaded at
    framebuffer points (fx, fy): coords = t * (uv0, 1) at the point and at the points one pixel right and one down, each through the
    triangle's own R6 weights; dpdx / dpdy their forward differences.  `depth_pass`: raw uv0 (no transform) and dpdy := dpdx, as
    depth.wgsl:108-110 writes it.  The error bound charges the f32 weights (vertex_reference.weight_error_bound), three roundings of
    each sum of products and the transform, doubled."""
    t = np.eye(3) if (t is None or depth_pass) else t
    pts, errs = [], []
    for ox, oy in ((0.0, 0.0), (1.0, 0.0), (0.0, 1.0)):
        nx, ny = vref.ndc(fx + ox, fy + oy, width, height)
        b, eb = vref.weights(xyw, nx, ny), vref.weight_error_bound(xyw, nx, ny)
        uv = b @ uv_tri
        e_uv = eb @ np.abs(uv_tri) + 3 * U * (np.abs(b) @ np.abs(uv_tri))
        c = uv @ t[:2, :2] + t[2, :2]
        e = e_uv @ np.abs(t[:2, :2]) + 3 * U * (np.abs(uv) @ np.abs(t[:2, :2]) + np.abs(t[2, :2]))
        pts.append(c)
        errs.append(2.0 * e.max(axis=1))
    c0, cx, cy = pts
    if depth_pass:
        cy, errs[2] = c0 + (cx - c0), errs[1]
    dx, dy = cx - c0, cy - c0
    ed = errs[0] + np.maximum(errs[1], errs[2]) + U * np.maximum(np.abs(dx).max(axis=1), np.abs(dy).max(axis=1))
    return TexCoords(c0[:, 0], c0[:, 1], dx[:, 0], dx[:, 1], dy[:, 0], dy[:, 1], errs[0], ed)


# ------------------------------------------------------------------ get_pixel_data_inner (opaque.wgsl:203-424)
@dataclass
class PixelInputs:
    """What get_pixel_data_inner hands to the lighting for N fragments, each with its error bound from the samples: albedo (N, 4),
    the tangent-space normal-map texel (N, 4) (None without a normal texture) and the scalar parameters (N,), emissive (N, 3)."""
    albedo: np.ndarray
    nmap: object
    ao: np.ndarray
    roughness: np.ndarray
    metallic: np.ndarray
    reflectance: np.ndarray
    clear_coat: np.ndarray
    cc_roughness: np.ndarray
    emissive: np.ndarray
    unlit: bool
    samples: dict           # slot -> Sampled, for the census and the bound


def pixel_data(rec, c: TexCoords, vcolor, table: Table):
    """get_pixel_data_inner branch for branch: `rec` the material record as the kernels read it, `c` the fragments' TexCoords,
    `vcolor` (N, 4) the interpolated vertex colour.  Returns (value, bound) PixelInputs pair: the second holds each field's bound."""
    flags = int(rec["flags"])
    tex = rec["textures"]
    linear = not (flags & MAT_NEAREST)
    f = lambda k: float(np.float32(rec[k]))
    n = len(c.u)
    samples = {}

    def read(slot):
        if tex[slot] == 0:
            return None
        if slot not in samples:
            samples[slot] = sample_slot(table, int(tex[slot]), linear, c)
        return samples[slot]

    def scaled(const, slot, ch):
        """material constant * texture channel (the constant where the slot is absent), and its bound."""
        s = read(slot)
        if s is None:
            return np.full(n, const), np.zeros(n)
        b = s.bound()
        return const * s.value[:, ch], abs(const) * b[:, ch]

    # albedo (:211-229)
    if flags & MAT_ALBEDO_ACTIVE:
        s = read(TEX_ALBEDO)
        alb, alb_b = (np.ones((n, 4)), np.zeros((n, 4))) if s is None else (s.value, s.bound())
        if flags & MAT_ALBEDO_BLEND:
            vc = np.concatenate([srgb_decode(vcolor[:, :3]) if flags & MAT_ALBEDO_VERTEX_SRGB else vcolor[:, :3], vcolor[:, 3:]], axis=1)
            alb, alb_b = alb * vc, alb_b * np.abs(vc)
    else:
        alb, alb_b = np.broadcast_to([0.0, 0.0, 0.0, 1.0], (n, 4)), np.zeros((n, 4))
    ma = np.asarray(rec["albedo"], dtype=np.float32).astype(np.float64)
    alb, alb_b = alb * ma, alb_b * np.abs(ma)
    unlit = bool(flags & MAT_UNLIT)
    nm = read(TEX_NORMAL) if not unlit else None
    nmap = None if nm is None else (nm.value, nm.bound())
    # AO, metallic, roughness (:280-351)
    if flags & MAT_AOMR_COMBINED:
        ao, rough, metal = scaled(f("ambient_occlusion"), TEX_ROUGHNESS, 0), scaled(f("roughness"), TEX_ROUGHNESS, 1), scaled(f("metallic"), TEX_ROUGHNESS, 2)
    elif flags & MAT_AOMR_BW_SPLIT:
        rough, metal, ao = scaled(f("roughness"), TEX_ROUGHNESS, 0), scaled(f("metallic"), TEX_METALLIC, 0), scaled(f("ambient_occlusion"), TEX_AMBIENT_OCCLUSION, 0)
    else:
        k = 1 if flags & MAT_AOMR_SWIZZLED_SPLIT else 0                      # .gb or .rg
        rough, metal = scaled(f("roughness"), TEX_ROUGHNESS, k), scaled(f("metallic"), TEX_ROUGHNESS, k + 1)
        ao = scaled(f("ambient_occlusion"), TEX_AMBIENT_OCCLUSION, 0)
    refl = scaled(f("reflectance"), TEX_REFLECTANCE, 0)                      # :355-359
    if flags & MAT_CC_GLTF_COMBINED:                                          # :363-390
        cc, ccr = scaled(f("clear_coat"), TEX_CLEAR_COAT, 0), scaled(f("clear_coat_roughness"), TEX_CLEAR_COAT, 1)
    else:
        cc = scaled(f("clear_coat"), TEX_CLEAR_COAT, 0)
        ccr = scaled(f("clear_coat_roughness"), TEX_CLEAR_COAT_ROUGHNESS, 1 if flags & MAT_CC_GLTF_SPLIT else 0)
    em_c = np.asarray(rec["emissive"], dtype=np.float32).astype(np.float64)   # :394-398
    s = read(TEX_EMISSIVE)
    em = (np.broadcast_to(em_c, (n, 3)), np.zeros((n, 3))) if s is None else (em_c * s.value[:, :3], np.abs(em_c) * s.bound()[:, :3])
    val = PixelInputs(alb, None if nmap is None else nmap[0], ao[0], rough[0], metal[0], refl[0], cc[0], ccr[0], em[0], unlit, samples)
    bnd = PixelInputs(alb_b, None if nmap is None else nmap[1], ao[1], rough[1], metal[1], refl[1], cc[1], ccr[1], em[1], unlit, samples)
    return val, bnd


FIELDS = (("albedo", 4), ("ao", 1), ("roughness", 1), ("metallic", 1), ("reflectance", 1), ("clear_coat", 1), ("cc_roughness", 1), ("emissive", 3))


def untextured_records(px: PixelInputs):
    """(N,) material records whose untextured fs_main (tests/shade_reference.py) sees the pixel data `px`: the albedo as the constant
    with only ALBEDO_ACTIVE (no vertex blend: it is already applied), the textured parameters as the constants."""
    n = len(px.ao)
    r = np.zeros(n, dtype=MATERIAL_DTYPE)
    r["albedo"], r["ambient_occlusion"], r["roughness"], r["metallic"] = px.albedo, px.ao, px.roughness, px.metallic
    r["reflectance"], r["clear_coat"], r["clear_coat_roughness"], r["emissive"] = px.reflectance, px.clear_coat, px.cc_roughness, px.emissive
    r["flags"] = MAT_ALBEDO_ACTIVE | (MAT_UNLIT if px.unlit else 0)
    return r


def fragment_normal(px: PixelInputs, flags, vnormal, vtangent):
    """:244-276: the normal map through the tangent basis, else the interpolated normal (fs_main normalises it)."""
    if px.nmap is None:
        return vnormal
    return vref.tbn_normal(vnormal, vtangent, vref.normal_map_value(px.nmap, flags))


def perturbed(px: PixelInputs, bnd: PixelInputs, field, ch, sign):
    """A copy of `px` with one channel of one field moved by its bound."""
    from dataclasses import replace
    a = np.array(getattr(px, field), dtype=np.float64, copy=True)
    b = getattr(bnd, field)
    if a.ndim == 1:
        a = a + sign * b
    else:
        a[:, ch] += sign * b[:, ch]
    return replace(px, **{field: a})


# ------------------------------------------------------------------ the cutout decisions
@dataclass
class Discard:
    discard: np.ndarray     # alpha < alpha_cutout
    near: np.ndarray        # the float64 alpha lies within its bound of alpha_cutout
    alpha: np.ndarray


def forward_discard(rec, c: TexCoords, vcolor, table: Table):
    """opaque.wgsl:231-235: the albedo alpha of get_pixel_data_inner (transformed coordinates, the material's sampler, vertex alpha
    never sRGB-decoded, material alpha) against alpha_cutout."""
    val, bnd = pixel_data(rec, c, vcolor, table)
    return _decide(val.albedo[:, 3], bnd.albedo[:, 3], rec)


def depth_discard(rec, c: TexCoords, valpha, table: Table):
    """depth.wgsl:104-126 with TexCoords from `coords(..., depth_pass=True)`: the linear sampler, alpha *= vertex alpha, then the
    material alpha, against alpha_cutout."""
    flags, slot = int(rec["flags"]), int(rec["textures"][TEX_ALBEDO])
    n = len(c.u)
    alpha, b = np.ones(n), np.zeros(n)
    if flags & MAT_ALBEDO_ACTIVE:
        if slot:
            s = sample_slot(table, slot, True, c)
            alpha, b = s.value[:, 3], s.bound()[:, 3]
        if flags & MAT_ALBEDO_BLEND:
            alpha, b = alpha * valpha, b * np.abs(valpha)
    ma = float(np.float32(rec["albedo"][3]))
    return _decide(alpha * ma, b * abs(ma), rec)


def _decide(alpha, b, rec):
    cut = float(np.float32(rec["alpha_cutout"]))
    return Discard(alpha < cut, np.abs(alpha - cut) <= b + 2 * U * np.abs(alpha), alpha)
