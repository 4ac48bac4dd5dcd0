"""fs_main of opaque.wgsl for untextured materials, restated in float64 numpy: the specification that the shading kernels
(rend3_b200/csrc/r3_shade.cu) and the oracle (oracle/r3_oracle_forward.inc) are both checked against.

Line numbers cite rend3-routine/shaders/src/opaque.wgsl unless another file is named.  WGSL min / max / saturate are IEEE
minNum / maxNum here (DESIGN.md §2): a NaN operand yields the other operand, which is np.fmin / np.fmax.  Every function takes
arrays over N fragments and evaluates each formula once, in float64, from the f32 values the kernels receive."""
import numpy as np

from rend3_b200.layouts import MAT_ALBEDO_ACTIVE, MAT_ALBEDO_BLEND, MAT_ALBEDO_VERTEX_SRGB, MAT_UNLIT

PI = 3.14159265359                 # math/consts.wgsl:1
TOL = 1e-4                         # tests/test_gpu_parity.py hdr_close: absolute below 1.0, relative above
PERTURB = 2.0 ** -20               # relative per-component perturbation of the sensitivity allowance


def saturate(x):                   # math/color.wgsl:21-23, clamp with minNum / maxNum
    return np.fmin(np.fmax(x, 0.0), 1.0)


def dot(a, b):
    return np.sum(a * b, axis=-1)


def normalize(a):
    return a / np.sqrt(dot(a, a))[..., None]


def srgb_to_linear(e):             # math/color.wgsl:3-9 (srgb_display_to_scene)
    return np.where(e > 0.04045, ((e + 0.055) / 1.055) ** 2.4, e / 12.92)


def f32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


class Pixel:
    """get_pixel_data_inner (:203-424) for a material without textures, per fragment.  `mat` is an (N,) array of MATERIAL_DTYPE
    records (PbrMaterial.to_record), `vcolor` the (N, 4) interpolated vertex colour, `normal` the (N, 3) interpolated normal."""

    def __init__(self, mat, vcolor, normal):
        flags = mat["flags"].astype(np.uint32)
        active = (flags & MAT_ALBEDO_ACTIVE) != 0
        blend = (flags & MAT_ALBEDO_BLEND) != 0
        srgb = (flags & MAT_ALBEDO_VERTEX_SRGB) != 0
        vc = np.concatenate([np.where(srgb[:, None], srgb_to_linear(vcolor[:, :3]), vcolor[:, :3]), vcolor[:, 3:]], axis=1)
        albedo = np.where(active[:, None], np.where(blend[:, None], vc, 1.0), np.array([0.0, 0.0, 0.0, 1.0]))   # :213-228
        self.albedo = albedo * f32(mat["albedo"])                                                               # :229
        self.unlit = (flags & MAT_UNLIT) != 0                                                                   # :239-242
        self.normal = normalize(normal)
        self.ao = f32(mat["ambient_occlusion"])                                                                 # :280-349, no textures
        metallic, reflectance = f32(mat["metallic"]), f32(mat["reflectance"])                                   # :353-357
        clear_coat, cc_rough = f32(mat["clear_coat"]), f32(mat["clear_coat_roughness"])                         # :361-388
        self.emissive = f32(mat["emissive"])                                                                    # :392-398
        self.diffuse = self.albedo[:, :3] * (1.0 - metallic)[:, None]                                           # :187-189,410
        dielectric = 0.16 * reflectance * reflectance                                                           # :195-197,413
        self.f0 = self.albedo[:, :3] * metallic[:, None] + (dielectric * (1.0 - metallic))[:, None]             # :191-193,414
        self.perceptual = clear_coat_remap(f32(mat["roughness"]), clear_coat, cc_rough)                         # :416-420
        self.roughness = self.perceptual * self.perceptual                                                      # :199-201,421


def clear_coat_remap(perceptual, clear_coat, cc_rough):
    """:416-420: mix(perceptual, max(perceptual, cc_rough), clear_coat) when clear_coat != 0."""
    mixed = perceptual * (1.0 - clear_coat) + np.fmax(perceptual, cc_rough) * clear_coat
    return np.where(clear_coat != 0.0, mixed, perceptual)


def surface_shading(l, intensity, px, v, occlusion, noh_scale=1.0):
    """:440-468 with math/brdf.wgsl:3-7 (GGX D), :9-11 (Schlick F), :24-26 (Lambert), :28-33 (correlated Smith V).  `noh_scale`
    lets the sensitivity allowance move n.h (see with_sensitivity)."""
    n = px.normal
    h = normalize(v + l)
    nov = np.abs(dot(n, v)) + 0.00001
    nol = saturate(dot(n, l))
    noh = saturate(dot(n, h)) * noh_scale
    loh = saturate(dot(l, h))
    f90 = saturate(np.sum(px.f0, axis=-1) * 16.5)                                                             # :449, 50 * 0.33
    a2 = px.roughness * px.roughness
    fd = (noh * a2 - noh) * noh + 1.0
    d = a2 / (PI * fd * fd)
    f = px.f0 + (f90[:, None] - px.f0) * ((1.0 - loh) ** 5)[:, None]
    vis = 0.5 / (nov * np.sqrt((-nol * a2 + nol) * nol + a2) + nol * np.sqrt((-nov * a2 + nov) * nov + a2))
    color = px.diffuse * (1.0 / PI) + (d * vis)[:, None] * f
    return (color * intensity) * (nol * occlusion)[:, None]


def point_attenuation(d, radius):
    """:536-539: s = saturate(d / radius), (1 - s^2)^2 / (1 + s^2).  0 at and beyond a positive radius; 1 for a negative or NaN
    radius (the ratio saturates to 0), and for radius 0 at d = 0."""
    s = saturate(d / radius)
    s2 = s * s
    return (1.0 - s2) ** 2 / (1.0 + s2)


def fs_main(vp, normal, mat, vcolor, ambient, dir_l=(), dir_color=(), shadow=None, pl_pos=(), pl_color=(), pl_radius=(), noh_scale=1.0):
    """:470-551 per fragment.  vp (N, 3) view position, dir_l (D, 3) the light vectors l = normalize(view_mat3 * -direction),
    dir_color (D, 3), shadow (N, D) the PCF factor (1 where there is no shadow), pl_pos / pl_color (P, 3) and pl_radius (P,) the
    point lights in view space.  Returns (N, 4)."""
    with np.errstate(all="ignore"):
        vp = np.asarray(vp, dtype=np.float64)
        px = Pixel(mat, np.asarray(vcolor, dtype=np.float64), np.asarray(normal, dtype=np.float64))
        v = -normalize(vp)                                                                                    # :481
        color = px.emissive.copy()                                                                            # :486
        for i in range(len(dir_l)):                                                                           # :487-522
            occ = px.ao * (1.0 if shadow is None else shadow[:, i])
            color += surface_shading(np.broadcast_to(f32(dir_l[i]), vp.shape), f32(dir_color[i]), px, v, occ, noh_scale)
        for i in range(len(pl_radius)):                                                                       # :524-546
            delta = f32(pl_pos[i]) - vp
            d = np.sqrt(dot(delta, delta))
            att = point_attenuation(d, np.float64(np.float32(pl_radius[i])))
            s = surface_shading(delta / d[:, None], f32(pl_color[i]) * att[:, None], px, v, px.ao, noh_scale)
            color += np.fmax(s, 0.0)
        amb = f32(ambient)
        lit = np.fmax(amb * px.albedo, np.concatenate([color, px.albedo[:, 3:]], axis=1))                    # :548-550
        return np.where(px.unlit[:, None], px.albedo, lit)                                                    # :476-478


def ggx_peak_margin(vp, normal, mat, pl_pos):
    """min over the point lights of 1 - noh^2 (1 - a^2), the denominator of brdf_d_ggx: where it is small (a roughness-0
    material facing a light's half vector) D is a 0 / 0 or huge, and only the NaN pattern is comparable."""
    with np.errstate(all="ignore"):
        vp = np.asarray(vp, dtype=np.float64)
        px = Pixel(mat, np.ones((len(vp), 4)), np.asarray(normal, dtype=np.float64))
        v = -normalize(vp)
        a2 = px.roughness ** 2
        out = np.full(len(vp), np.inf)
        for p in pl_pos:
            delta = f32(p) - vp
            h = normalize(v + normalize(delta))
            noh = saturate(dot(px.normal, h))
            out = np.fmin(out, 1.0 - noh * noh * (1.0 - a2))
        return out


def with_sensitivity(vp, normal, pl_pos, fn, rel=PERTURB):
    """fn(vp, normal, pl_pos, noh_scale) and the largest change of it when the view position, the normal and the point-light
    positions are each perturbed by `rel` relative per component, either sign, and when n.h moves down by `rel` relative.  The
    first three carry the f32 input rounding through the BRDF.  The last is needed at the GGX peak, where the first-order change
    vanishes but the error of n.h itself (normalisations with rsqrt approximations on the kernel's side) is amplified by 1/a^2."""
    vp, normal = np.asarray(vp, dtype=np.float64), np.asarray(normal, dtype=np.float64)
    pl_pos = np.asarray(pl_pos, dtype=np.float64).reshape(-1, 3)
    base = fn(vp, normal, pl_pos, 1.0)
    with np.errstate(invalid="ignore"):
        sens = np.abs(fn(vp, normal, pl_pos, 1.0 - rel) - base)
        for which in range(3 if len(pl_pos) else 2):
            for axis in range(3):
                for sign in (-1.0, 1.0):
                    args = [vp.copy(), normal.copy(), pl_pos.copy()]
                    args[which][:, axis] *= 1.0 + sign * rel
                    sens = np.fmax(sens, np.abs(fn(*args, 1.0) - base))
    return base, sens


def compare(got, want, sens, mask=None, f16=False):
    """Channel values of `got` against the float64 `want`: the bound is TOL (relative above 1.0) plus the sensitivity `sens`
    (plus one half-precision ulp when the value went through an rgba16f target).  Both NaN counts as equal.  Returns
    (bad mask, number of values checked, fraction of the checked values that needed more than TOL)."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    if mask is None:
        mask = np.ones(want.shape[:-1], dtype=bool)
    m = np.broadcast_to(mask[..., None], want.shape) & np.isfinite(want)
    scale = np.maximum(1.0, np.abs(want))
    err = np.abs(got - want)
    base_bound = TOL * scale + (np.maximum(np.abs(want) * 2.0 ** -10, 2.0 ** -24) if f16 else 0.0)
    bound = base_bound + sens
    bad = m & ~(np.nan_to_num(err, nan=np.inf) <= bound)
    n = int(np.count_nonzero(m))
    needed = np.count_nonzero(m & (np.nan_to_num(err, nan=np.inf) > base_bound))
    return bad, n, (needed / n if n else 0.0)


def directional_shadow(vp, lm, offset, size, inv_res, atlas):
    """The shadow factor of one directional light (:491-516) from the shadow atlas (H, W): shadow-space position lm * (vp, 1)
    (lm = light.view_proj * inv_view, column-major), atlas coordinates mix(top_left, top_right, (x, 1 - y)), PCF5 where the literal
    any() region test and 0 <= z <= 1 pass, else exactly 1.  Returns (factor, margin, sampled): margin is the smallest distance of
    a compared texel or of a region-test operand from its decision, inf where a decision cannot flip."""
    vp = np.asarray(vp, dtype=np.float64)
    m = f32(lm).reshape(4, 4)                                                    # m[column][row]
    sn = vp @ m[:3] + m[3]
    flx, fly, snz = sn[:, 0] * 0.5 + 0.5, sn[:, 1] * 0.5 + 0.5, sn[:, 2]          # :491-493
    off, sz, inv = f32(offset), f32(size), f32(inv_res)
    cu = off[0] * (1.0 - flx) + (off[0] + sz[0]) * flx                           # :496-498, mix
    cv = off[1] * fly + (off[1] + sz[1]) * (1.0 - fly)
    tl, tr = off + inv * 1.5, off + sz - inv * 1.5                               # :504-506
    sampled = ((flx >= tl[0]) | (fly >= tl[1])) & ((flx <= tr[0]) | (fly <= tr[1])) & (snz >= 0.0) & (snz <= 1.0)   # :509-514
    factor, margin = pcf5(atlas, cu, cv, snz)
    edge = np.min(np.abs(np.stack([flx - tl[0], fly - tl[1], flx - tr[0], fly - tr[1], snz, snz - 1.0])), axis=0)
    return np.where(sampled, factor, 1.0), np.minimum(np.where(sampled, margin, np.inf), edge), sampled


def pcf5(atlas, u, v, ref):
    """shadow/pcf.wgsl:1-9 on an atlas (H, W) in float64: five textureSampleCompareLevel taps at texel offsets (0,0), (0,1),
    (0,-1), (1,0), (-1,0), each the bilinear weight of four GreaterEqual compares with Repeat addressing.  Returns (factor,
    margin): margin is the smallest |ref - texel| over the 20 compared texels, so a caller can exclude near-ties."""
    atlas = np.asarray(atlas, dtype=np.float64)
    h, w = atlas.shape
    u, v, ref = (np.asarray(a, dtype=np.float64) for a in (u, v, ref))
    total = np.zeros_like(ref)
    margin = np.full_like(ref, np.inf)
    for ox, oy in ((0, 0), (0, 1), (0, -1), (1, 0), (-1, 0)):
        x, y = u * w + ox - 0.5, v * h + oy - 0.5
        x0, y0 = np.floor(x), np.floor(y)
        fx, fy = x - x0, y - y0
        tap = np.zeros_like(ref)
        for dx, dy, wt in ((0, 0, (1 - fx) * (1 - fy)), (1, 0, fx * (1 - fy)), (0, 1, (1 - fx) * fy), (1, 1, fx * fy)):
            t = atlas[((y0 + dy).astype(np.int64) % h), ((x0 + dx).astype(np.int64) % w)]
            tap += np.where(ref >= t, 1.0, 0.0) * wt
            margin = np.minimum(margin, np.abs(ref - t))
        total += tap
    return total * 0.2, margin
