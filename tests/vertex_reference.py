"""The vertex stage of opaque.wgsl restated in float64 numpy: get_vertices' defaults, vs_main's attribute half, the
perspective-correct interpolation of raster rule R6 and the tangent basis of a normal map.  What it produces is what fs_main
receives (view position, normal, vertex colour); tests/shade_reference.py's fs_main takes it from there.

Line numbers cite rend3-routine/shaders/src/opaque.wgsl unless another file is named.  Inputs are the f32 values the kernels
receive (the MV / MVP bits of readback_object_matrices, the mesh's attribute arrays); every formula is evaluated once, in
float64.  Matrices are column-major, m[column][row], like glam and the object-matrix records."""
import numpy as np

from rend3_b200.layouts import MAT_BICOMPONENT_NORMAL, MAT_SWIZZLED_NORMAL, MAT_YDOWN_NORMAL
from shade_reference import normalize


def columns(m16):
    """A 16-float column-major matrix as float64 m[column][row]."""
    return np.asarray(m16, dtype=np.float32).astype(np.float64).reshape(4, 4)


# ------------------------------------------------------------------ get_vertices (rend3/src/shader.rs:249-316)
def unpack_colour(rgba8, n):
    """vertex colour 0: unpack4x8unorm of the attribute word, byte 0 = r (vertex_attributes.wgsl:82-85,
    rend3-types/src/attribute.rs:125-135).  `rgba8` is the (n, 4) uint8 attribute in memory order; absent (None) is vec4(1.0)."""
    if rgba8 is None:
        return np.ones((n, 4))
    words = np.ascontiguousarray(rgba8, dtype=np.uint8).reshape(n, 4).view(np.uint32).reshape(n)
    return np.stack([((words >> (8 * k)) & 0xFF).astype(np.float64) / 255.0 for k in range(4)], axis=1)


def attribute(a, n, width):
    """A float attribute as float64 (n, width); an absent tangent or uv0 reads as zero."""
    if a is None:
        return np.zeros((n, width))
    return np.asarray(a, dtype=np.float32).astype(np.float64).reshape(n, width)


# ------------------------------------------------------------------ vs_main (:114-134)
def inv_scale_squared(mv):
    """math/matrix.wgsl:1-7 on mv3 = the xyz of MV's columns 0-2 (:118): 1 / dot(column, column) per COLUMN.  For a matrix whose
    columns are not orthogonal (a shear) mv3 * (inv_scale_sq * n) is not the inverse transpose applied to n; the WGSL is the
    specification, so this follows it literally.  IEEE: a zero column gives 1 / 0 = inf."""
    m = columns(mv)[:3, :3]
    with np.errstate(divide="ignore"):
        return 1.0 / np.sum(m * m, axis=1)


def transform_direction(mv, d, iss=True):
    """normalize(mv3 * (inv_scale_sq * d)) (:126-128) for (n, 3) directions; `iss=False` drops inv_scale_sq (for the census)."""
    m = columns(mv)[:3, :3]
    s = inv_scale_squared(mv) if iss else np.ones(3)
    with np.errstate(all="ignore"):
        sd = d * s                                  # inf * 0 = NaN where a column is zero
        return normalize(sd @ m)                    # sum over columns c of m[c] * sd[c]; normalize(0) = NaN


def vs_main(mv, pos, normal, tangent, iss=True):
    """(view_position (n, 4), normal (n, 3), tangent (n, 3)) of vs_out for float64 attribute arrays."""
    m = columns(mv)
    vp = np.concatenate([pos, np.ones((len(pos), 1))], axis=1) @ m          # model_view * vec4(pos, 1) (:124)
    return vp, transform_direction(mv, normal, iss), transform_direction(mv, tangent, iss)


def clip_xyw(mvp, pos):
    """clip.xyw = (model_view_proj * vec4(pos, 1)).xyw (:132) of the unclipped vertices."""
    c = np.concatenate([pos, np.ones((len(pos), 1))], axis=1) @ columns(mvp)
    return c[:, [0, 1, 3]], c[:, 2]


# ------------------------------------------------------------------ rule R6
def ndc(fx, fy, width, height):
    """Framebuffer position (pixels, y down) -> (ndc_x, ndc_y)."""
    return fx / (width * 0.5) - 1.0, 1.0 - fy / (height * 0.5)


def edge_values(xyw, nx, ny):
    """E_i = cross(p_j, p_k) . (ndc_x, ndc_y, 1) for a triangle's clip xyw (3, 3) at points (m,): (m, 3).  E_i = lambda_i det / w,
    with lambda the barycentric weights of the point in the triangle's plane and w its clip w."""
    q = np.stack([np.asarray(nx, dtype=np.float64), np.asarray(ny, dtype=np.float64), np.ones(np.shape(nx))], axis=-1)
    c = np.stack([np.cross(xyw[(i + 1) % 3], xyw[(i + 2) % 3]) for i in range(3)])     # (3, 3): c[i] = cross(p_j, p_k)
    return q @ c.T


def weights(xyw, nx, ny):
    """R6: b_i = E_i / sum(E) at (ndc_x, ndc_y), from the UNCLIPPED clip xyw, for points anywhere in the plane: outside the
    triangle (a 4x sample's primitive shaded at a pixel centre it does not cover) some weights are negative."""
    e = edge_values(xyw, nx, ny)
    with np.errstate(all="ignore"):
        return e / np.sum(e, axis=-1, keepdims=True)


U32 = 2.0 ** -24


def weight_error_bound(xyw, nx, ny):
    """A forward bound of the f32 rounding of R6's weights as the kernels evaluate them (cross products, the dot with
    (ndc_x, ndc_y, 1) in source order, the sum and the divisions, and ndc itself): (m, 3).  Next to a large triangle, or one whose
    vertices are close together relative to their clip coordinates, the cross products cancel, so the weights carry far more than
    one rounding.  Six roundings per path are charged, a few more than the longest path takes."""
    nx, ny = np.asarray(nx, dtype=np.float64), np.asarray(ny, dtype=np.float64)
    g = 6.0 * U32
    errs, es = [], []
    for i in range(3):
        a, b = xyw[(i + 1) % 3], xyw[(i + 2) % 3]
        c = np.cross(a, b)
        t = np.array([abs(a[1] * b[2]) + abs(a[2] * b[1]), abs(a[2] * b[0]) + abs(a[0] * b[2]), abs(a[0] * b[1]) + abs(a[1] * b[0])])
        dn = 2.0 * U32 * (1.0 + np.abs(nx)), 2.0 * U32 * (1.0 + np.abs(ny))     # ndc = f / (size / 2) - 1: two roundings
        errs.append(g * (t[0] * np.abs(nx) + t[1] * np.abs(ny) + t[2] + np.abs(c[0] * nx) + np.abs(c[1] * ny)) + np.abs(c[0]) * dn[0] + np.abs(c[1]) * dn[1])
        es.append(c[0] * nx + c[1] * ny + c[2])
    e, err = np.stack(es, axis=-1), np.stack(errs, axis=-1)
    s = np.sum(e, axis=-1, keepdims=True)
    err_s = np.sum(err, axis=-1, keepdims=True) + 2.0 * U32 * np.sum(np.abs(e), axis=-1, keepdims=True)
    with np.errstate(all="ignore"):
        b = e / s
        return (err + np.abs(b) * err_s) / np.abs(s) + U32 * np.abs(b)


# ------------------------------------------------------------------ the tangent basis (:244-276)
def normal_map_value(t, flags):
    """The tangent-space normal from the sampled texel t (m, 4): tri-component normalize(t.rgb * 2 - 1); bicomponent (t.rg, or
    t.ag when swizzled) * 2 - 1 with z = sqrt((1 - x^2) - y^2); y negated for a y-down map."""
    t = np.asarray(t, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        if flags & MAT_BICOMPONENT_NORMAL:
            xy = np.stack([t[:, 3] if flags & MAT_SWIZZLED_NORMAL else t[:, 0], t[:, 1]], axis=1) * 2.0 - 1.0
            n = np.concatenate([xy, np.sqrt((1.0 - xy[:, :1] ** 2) - xy[:, 1:] ** 2)], axis=1)
        else:
            n = normalize(t[:, :3] * 2.0 - 1.0)
    if flags & MAT_YDOWN_NORMAL:
        n = n * np.array([1.0, -1.0, 1.0])
    return n


def tbn_normal(vnormal, vtangent, nmap):
    """tbn * normal with tbn = mat3x3(normalize(tangent), cross(normalize(normal), normalize(tangent)), normalize(normal)); fs_main
    normalises the result (pixel.normal, :276).  NaN propagates: a zero tangent normalises to NaN."""
    with np.errstate(all="ignore"):
        n, t = normalize(vnormal), normalize(vtangent)
        b = np.cross(n, t)
        return t * nmap[:, :1] + b * nmap[:, 1:2] + n * nmap[:, 2:]
