"""Rule R13 (DESIGN.md §2) restated in numpy float32, one IEEE operation at a time: the directional light's shadow camera of
directional/shadow_camera.rs:6-33 and the light record of directional.rs:135-156.

The CUDA kernel (rend3_b200/csrc/r3_lights.cu) and the C oracle (oracle/r3_oracle_lights.c) follow the same steps; the tests hold the
three to each other bit for bit (any NaN equal to any NaN).  Every value is an np.float32 scalar and every step one operation on two of
them, so numpy rounds after each operation and never contracts."""
from __future__ import annotations

import numpy as np

from rend3_b200.layouts import CAMERA_HEADER_DTYPE, DIRECTIONAL_LIGHT_DTYPE, LIGHT_SOURCE_DTYPE, PCU_POSITIVE_AREA_VISIBLE

f32 = np.float32
ONE, ZERO, HALF = f32(1.0), f32(0.0), f32(0.5)


def dot3(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def cross(a, b):
    return (a[1] * b[2] - b[1] * a[2], a[2] * b[0] - b[2] * a[0], a[0] * b[1] - b[0] * a[1])


def normalize(a):
    r = ONE / np.sqrt(dot3(a, a))
    return (a[0] * r, a[1] * r, a[2] * r)


def look_to_lh(eye, d):
    """glam.py::look_to_lh with up = Y; m[c][r]."""
    up = (ZERO, ONE, ZERO)
    f = normalize(d)
    s = normalize(cross(up, f))
    u = cross(f, s)
    return [[s[0], u[0], f[0], ZERO], [s[1], u[1], f[1], ZERO], [s[2], u[2], f[2], ZERO], [-dot3(eye, s), -dot3(eye, u), -dot3(eye, f), ONE]]


def look_at(eye, center, lh):
    """look_at_lh: look_to_lh(eye, center - eye); look_at_rh (glam.py): look_to_lh(eye, eye - center)."""
    d = tuple(center[k] - eye[k] for k in range(3)) if lh else tuple(eye[k] - center[k] for k in range(3))
    return look_to_lh(eye, d)


def transform_point3(m, p):
    return tuple(((m[0][k] * p[0] + m[1][k] * p[1]) + m[2][k] * p[2]) + m[3][k] for k in range(3))


def inverse(m):
    """glam's SSE2 Mat4::inverse (GLM's cofactor expansion): coefficients a*b - c*d, cofactor columns ((v f - v f) + v f) times the sign
    vectors, det = (d.x + d.z) + (d.y + d.w) (SSE2 dot4), every element times 1 / det."""
    rows = [(2, 3), (1, 3), (1, 2), (0, 3), (0, 2), (0, 1)]
    fac = []
    for i, j in rows:
        c0 = m[2][i] * m[3][j] - m[3][i] * m[2][j]
        c2 = m[1][i] * m[3][j] - m[3][i] * m[1][j]
        c3 = m[1][i] * m[2][j] - m[2][i] * m[1][j]
        fac.append((c0, c0, c2, c3))
    vec = [(m[1][r], m[0][r], m[0][r], m[0][r]) for r in range(4)]
    terms = [(1, 0, 2, 1, 3, 2), (0, 0, 2, 3, 3, 4), (0, 1, 1, 3, 3, 5), (0, 2, 1, 4, 2, 5)]
    sign_a, sign_b = (ONE, -ONE, ONE, -ONE), (-ONE, ONE, -ONE, ONE)
    inv = []
    for c, (a, p, b, q, e, t) in enumerate(terms):
        sg = sign_b if c & 1 else sign_a
        inv.append([((vec[a][k] * fac[p][k] - vec[b][k] * fac[q][k]) + vec[e][k] * fac[t][k]) * sg[k] for k in range(4)])
    d = [m[0][k] * inv[k][0] for k in range(4)]
    rcp = ONE / ((d[0] + d[2]) + (d[1] + d[3]))
    return [[inv[c][k] * rcp for k in range(4)] for c in range(4)]


def orthographic(distance, lh):
    """orthographic_{lh,rh}(-h, h, -h, h, h, -h), h = distance * 0.5 (camera.rs:90-96, glam.py)."""
    half = distance * HALF
    left, right, bottom, top, near, far = -half, half, -half, half, half, -half
    rcp_w = ONE / (right - left)
    rcp_h = ONE / (top - bottom)
    r = ONE / (far - near) if lh else ONE / (near - far)
    return [[rcp_w + rcp_w, ZERO, ZERO, ZERO], [ZERO, rcp_h + rcp_h, ZERO, ZERO], [ZERO, ZERO, r, ZERO],
            [-(left + right) * rcp_w, -(top + bottom) * rcp_h, (-r) * near if lh else r * near, ONE]]


def mul(a, b):
    """glam.mul: column j = ((a0 b.x + a1 b.y) + a2 b.z) + a3 b.w."""
    return [[((a[0][k] * b[j][0] + a[1][k] * b[j][1]) + a[2][k] * b[j][2]) + a[3][k] * b[j][3] for k in range(4)] for j in range(4)]


def frustum(vp):
    """Frustum::from_matrix (world.py::frustum_from_matrix): left r3 + r0, right r3 - r0, top r3 - r1, bottom r3 + r1, near r3 - r2,
    each divided by |abc|."""
    out = []
    for r, plus in ((0, True), (0, False), (1, False), (1, True), (2, False)):
        q = [vp[c][3] + vp[c][r] if plus else vp[c][3] - vp[c][r] for c in range(4)]
        mag = np.sqrt(dot3(q, q))
        out.append([q[c] / mag for c in range(4)])
    return out


def shadow_camera(direction, distance, resolution, location, lh):
    """(view, view_proj, frustum) of one light, as nested lists of np.float32."""
    with np.errstate(all="ignore"):
        dr = tuple(f32(v) for v in direction)
        d = f32(distance)
        loc = tuple(f32(v) for v in location)
        texel = d / f32(resolution)
        origin_view = look_at((ZERO, ZERO, ZERO), dr, lh)
        cov = transform_point3(origin_view, loc)
        shadow_loc = (cov[0] - np.fmod(cov[0], texel), cov[1] - np.fmod(cov[1], texel), cov[2] - ZERO)
        new_loc = transform_point3(inverse(origin_view), shadow_loc)
        center = tuple(new_loc[k] + dr[k] for k in range(3))
        view = look_at(new_loc, center, lh)
        vp = mul(orthographic(d, lh), view)
        return view, vp, frustum(vp)


def evaluate(sources: np.ndarray, atlas_w: int, atlas_h: int, location, left_handed: bool):
    """(CAMERA_HEADER_DTYPE array with object_count 0, DIRECTIONAL_LIGHT_DTYPE array) for LIGHT_SOURCE_DTYPE records."""
    n = len(sources)
    heads = np.zeros(n, dtype=CAMERA_HEADER_DTYPE)
    lights = np.zeros(n, dtype=DIRECTIONAL_LIGHT_DTYPE)
    w, h = f32(atlas_w), f32(atlas_h)
    with np.errstate(all="ignore"):
        for i, s in enumerate(sources):
            view, vp, fr = shadow_camera(s["direction"], s["distance"], int(s["resolution"]), location, left_handed)
            heads[i]["view"] = np.array(view, dtype=f32).reshape(16)
            heads[i]["view_proj"] = np.array(vp, dtype=f32).reshape(16)
            heads[i]["frustum"] = np.array(fr, dtype=f32)
            heads[i]["shadow_index"] = i
            heads[i]["resolution"] = (f32(int(s["size"])), f32(int(s["size"])))
            heads[i]["flags"] = PCU_POSITIVE_AREA_VISIBLE if left_handed else 0
            lights[i]["view_proj"] = heads[i]["view_proj"]
            lights[i]["color"] = [f32(s["color"][k]) * f32(s["intensity"]) for k in range(3)]
            lights[i]["direction"] = s["direction"]
            lights[i]["inv_resolution"] = (ONE / w, ONE / h)
            lights[i]["atlas_offset"] = (f32(int(s["offset"][0])) / w, f32(int(s["offset"][1])) / h)
            lights[i]["atlas_size"] = (f32(int(s["size"])) / w, f32(int(s["size"])) / h)
    return heads, lights


def sources(rows):
    """rows: (direction, distance, resolution); placements packed along the atlas' first row, 64 texels each."""
    s = np.zeros(len(rows), dtype=LIGHT_SOURCE_DTYPE)
    for i, (d, dist, res) in enumerate(rows):
        s[i] = ((1.0, 0.9, 0.8), 1.0 + 0.5 * i, d, dist, res, (64 * i, 0), 64)
    return s
