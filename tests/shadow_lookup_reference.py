"""The directional shadow lookup of fs_main restated in float32, operation by operation in source order: opaque.wgsl:491-516 and
shadow/pcf.wgsl:1-9 as the oracle evaluates them (oracle/r3_oracle_forward.inc, fragment_stage and shadow_sample_pcf5).

Every value is a numpy float32 array and every operation rounds once, so on a fragment whose view position is the oracle's the
result equals the oracle's bit for bit, near-ties included.  The view position comes from `view_position`, raster rule R6 in the
oracle's order (shade_at_pixel).  Besides the factor, `lookup` returns each tap's texel coordinates, fractions and compared texel
values, so that a test can name the first value in the chain where two implementations part."""
import numpy as np

F = np.float32


def mat_point(m, p):
    """m (16,) column-major times (p, 1), accumulated x, y, z, w in the oracle's order (mat_point)."""
    m = np.asarray(m, dtype=F)
    p = np.asarray(p, dtype=F)
    r = [m[k] * p[..., 0] for k in range(4)]
    r = [r[k] + m[4 + k] * p[..., 1] for k in range(4)]
    r = [r[k] + m[8 + k] * p[..., 2] for k in range(4)]
    return np.stack([r[k] + m[12 + k] for k in range(4)], axis=-1)


def mat_vec(m, v):
    """m (16,) column-major times v (..., 4) (mat_vec)."""
    m = np.asarray(m, dtype=F)
    v = np.asarray(v, dtype=F)
    r = [m[k] * v[..., 0] for k in range(4)]
    for c in range(1, 4):
        r = [r[k] + m[4 * c + k] * v[..., c] for k in range(4)]
    return np.stack(r, axis=-1)


def mat_mul(a, b):
    """Column j of a * b is a * b[j] (mat_mul): lm = light.view_proj * uniforms.inv_view."""
    b = np.asarray(b, dtype=F).reshape(4, 4)
    return np.concatenate([mat_vec(a, b[j]) for j in range(4)])


def view_position(px, py, width, height, clip, view):
    """R6 at the centres of pixels (px, py) (arrays) for triangles whose three vertices have clip positions `clip` (..., 3, 4)
    and view positions `view` (..., 3, 4): perspective weights b (3 arrays) from the cross products of (x, y, w), and the
    interpolated view position (b0 * v0 + b1 * v1) + b2 * v2.  Returns (view position, b)."""
    hw, hh = F(width) * F(0.5), F(height) * F(0.5)
    nx = (np.asarray(px, dtype=F) + F(0.5)) / hw - F(1.0)
    ny = F(1.0) - (np.asarray(py, dtype=F) + F(0.5)) / hh
    p = [np.asarray(clip, dtype=F)[..., k, :] for k in range(3)]

    def cross_term(a, b):   # ((c.x * nx + c.y * ny) + c.z) with c = cross(a, b) over (x, y, w)
        cx, cy, cz = a[..., 1] * b[..., 3] - a[..., 3] * b[..., 1], a[..., 3] * b[..., 0] - a[..., 0] * b[..., 3], a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]
        return (cx * nx + cy * ny) + cz
    b = [cross_term(p[1], p[2]), cross_term(p[2], p[0]), cross_term(p[0], p[1])]
    s = (b[0] + b[1]) + b[2]
    b = [bk / s for bk in b]
    return interpolate(b, view), b


def interpolate(b, attr):
    """(b0 * a0 + b1 * a1) + b2 * a2 for a vertex attribute `attr` (..., 3, k)."""
    a = np.asarray(attr, dtype=F)
    return (b[0][..., None] * a[..., 0, :] + b[1][..., None] * a[..., 1, :]) + b[2][..., None] * a[..., 2, :]


def normalize3(a):
    """a / sqrt((x * x + y * y) + z * z) per component (normalize3 of the oracle)."""
    a = np.asarray(a, dtype=F)
    n = np.sqrt((a[..., 0] * a[..., 0] + a[..., 1] * a[..., 1]) + a[..., 2] * a[..., 2])
    return a / n[..., None]


def dot3(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


TAPS = ((0, 0), (0, 1), (0, -1), (1, 0), (-1, 0))   # shadow/pcf.wgsl:1-9, summed in this order


class Lookup:
    """One directional light's lookup at N fragments.  factor (N,) is 1 where the lookup is skipped; sn (N, 4), flx, fly, cu, cv,
    the region bounds and `sampled` are the chain up to the sampler; per tap t (5 of them): x[t], y[t] (the texel-space
    coordinates), fx[t], fy[t], ix[t], iy[t] (the unwrapped floor), texels[t] (N, 4) in the order (x0,y0) (x1,y0) (x0,y1) (x1,y1)
    after the Repeat wrap, and tap[t], the bilinear result."""


def lookup(vp, lm, offset, size, inv_res, atlas):
    vp = np.asarray(vp, dtype=F)
    atlas = np.asarray(atlas, dtype=F)
    H, W = atlas.shape
    o = Lookup()
    o.sn = sn = mat_vec(lm, vp)                                                 # :491
    o.flx = flx = sn[:, 0] * F(0.5) + F(0.5)
    o.fly = fly = sn[:, 1] * F(0.5) + F(0.5)
    locy = F(1.0) - fly
    tlx, tly = F(offset[0]), F(offset[1])
    trx, try_ = tlx + F(size[0]), tly + F(size[1])
    o.cu = cu = tlx * (F(1.0) - flx) + trx * flx                               # mix(top_left, top_right, (x, 1 - y))
    o.cv = cv = tly * (F(1.0) - locy) + try_ * locy
    bx, by = F(inv_res[0]) * F(1.5), F(inv_res[1]) * F(1.5)
    o.bounds = (tlx + bx, tly + by, trx - bx, try_ - by)
    tl_x, tl_y, tr_x, tr_y = o.bounds
    snz = sn[:, 2]
    # the literal any() of :509-514: x OR y inside each bound
    o.sampled = ((flx >= tl_x) | (fly >= tl_y)) & ((flx <= tr_x) | (fly <= tr_y)) & (snz >= F(0.0)) & (snz <= F(1.0))
    o.x, o.y, o.fx, o.fy, o.ix, o.iy, o.texels, o.tap = [], [], [], [], [], [], [], []
    wf, hf = F(W), F(H)
    with np.errstate(invalid="ignore", over="ignore"):
        r = np.zeros(len(vp), dtype=F)
        for ox, oy in TAPS:
            x = (cu * wf + F(ox)) - F(0.5)
            y = (cv * hf + F(oy)) - F(0.5)
            x0, y0 = np.floor(x), np.floor(y)
            fx, fy = x - x0, y - y0
            ok = np.isfinite(x0) & np.isfinite(y0)
            ix = np.where(ok, x0, 0).astype(np.int64)
            iy = np.where(ok, y0, 0).astype(np.int64)
            xs, ys = (ix % W, (ix + 1) % W), (iy % H, (iy + 1) % H)
            t = np.stack([atlas[ys[0], xs[0]], atlas[ys[0], xs[1]], atlas[ys[1], xs[0]], atlas[ys[1], xs[1]]], axis=1)
            c = np.where(snz[:, None] >= t, F(1.0), F(0.0))                    # GreaterEqual
            gx = F(1.0) - fx
            top = c[:, 0] * gx + c[:, 1] * fx
            bot = c[:, 2] * gx + c[:, 3] * fx
            tap = top * (F(1.0) - fy) + bot * fy
            r = r + tap
            for lst, val in ((o.x, x), (o.y, y), (o.fx, fx), (o.fy, fy), (o.ix, ix), (o.iy, iy), (o.texels, t), (o.tap, tap)):
                lst.append(val)
        o.pcf = r * F(0.2)
    o.factor = np.where(o.sampled, o.pcf, F(1.0)).astype(F)
    return o


def near_ties(o, ulps=4):
    """(N,) True where some compare of a sampled fragment is within `ulps` float32 ulps of its reference depth."""
    snz = o.sn[:, 2]
    tol = ulps * np.spacing(np.abs(snz).astype(F))
    near = np.zeros(len(snz), dtype=bool)
    for t in o.texels:
        near |= (np.abs(snz[:, None].astype(np.float64) - t.astype(np.float64)) <= tol[:, None]).any(axis=1)
    return near & o.sampled


def describe(o, i, light):
    """The chain of fragment i for light `light`: what a failing test prints."""
    s = [f"light {light}: sn = {o.sn[i].tolist()} (snz = {float(o.sn[i, 2])!r}), flx = {float(o.flx[i])!r}, fly = {float(o.fly[i])!r}, "
         f"cu = {float(o.cu[i])!r}, cv = {float(o.cv[i])!r}, sampled = {bool(o.sampled[i])}"]
    for t, (ox, oy) in enumerate(TAPS):
        s.append(f"  tap ({ox:+d},{oy:+d}): x = {float(o.x[t][i])!r}, y = {float(o.y[t][i])!r}, floor = ({int(o.ix[t][i])}, {int(o.iy[t][i])}), "
                 f"fx = {float(o.fx[t][i])!r}, fy = {float(o.fy[t][i])!r}, texels = {o.texels[t][i].tolist()}, tap = {float(o.tap[t][i])!r}")
    return "\n".join(s)
