"""Skybox scenes: six solid-colour faces seen through a 90-degree camera at the origin looking down an axis — the whole target shows
that face — a labelled cube for the (s, t) orientation of rule R10 (texel = (column, row, face, 1)), random cubes in every sky
format, and the views of tests/test_skybox_reference.py: random rotations with roll, orthographic and raw projections, and exact
permutation views whose diagonal pixels tie two axes bit for bit."""
from dataclasses import dataclass
from typing import Tuple

import numpy as np

from rend3_b200 import glam
from rend3_b200.routines import BaseRenderGraphSettings, frame_uniforms
from rend3_b200.runner import TestRunner
from rend3_b200.world import BLEND, LEFT, Camera, PbrMaterial

import skybox_reference as sref

FACE_COLOURS = np.array([[255, 0, 0, 255], [0, 255, 0, 255], [0, 0, 255, 255], [255, 255, 0, 255], [0, 255, 255, 255], [255, 0, 255, 255]], dtype=np.uint8)
# looking along +X, -X, +Y, -Y, +Z, -Z (up vectors chosen so that look_at is well defined)
LOOK = [((1, 0, 0), (0, 1, 0)), ((-1, 0, 0), (0, 1, 0)), ((0, 1, 0), (0, 0, -1)), ((0, -1, 0), (0, 0, 1)), ((0, 0, 1), (0, 1, 0)), ((0, 0, -1), (0, 1, 0))]


def solid_faces(size=8):
    return [np.broadcast_to(FACE_COLOURS[f], (size, size, 4)).copy() for f in range(6)]


def build(backend, faces, face_index, srgb=False, mips="generated"):
    r = TestRunner(backend, LEFT)
    r.renderer.set_skybox(faces, srgb=srgb, mips=mips)
    direction, up = LOOK[face_index]
    view = glam.look_at_lh(np.zeros(3, dtype=np.float32), np.array(direction, dtype=np.float32), np.array(up, dtype=np.float32))
    r.renderer.set_aspect_ratio(1.0)
    r.renderer.set_camera_data(Camera(("perspective", 90.0, 0.1), view))
    return r


# ------------------------------------------------------------------ cubes
def labelled_faces(n):
    """RGBA32F faces whose texel is (column, row, face, 1): a sample names the texel it read."""
    row, col = np.mgrid[0:n, 0:n].astype(np.float32)
    return [np.stack([col, row, np.full_like(col, f), np.ones_like(col)], axis=-1) for f in range(6)]


def random_faces(n, fmt, seed):
    """Six random faces: "rgba8" / "rgba8_srgb" texels, or "rgba32f" values of either sign up to 1e5 with a few +-inf and NaN texels
    (NaN in red, infinities in green, on the -X and +Y faces only, so that the other channels and faces keep finite values)."""
    rng = np.random.default_rng(seed)
    if fmt != "rgba32f":
        return [rng.integers(0, 256, (n, n, 4), dtype=np.uint8) for _ in range(6)]
    faces = []
    for f in range(6):
        v = (rng.choice([-1.0, 1.0], (n, n, 4)) * 10.0 ** rng.uniform(-3, 5, (n, n, 4))).astype(np.float32)
        if f in (1, 2) and n >= 3:
            k = max(1, n * n // 64)
            idx = rng.choice(n * n, 3 * k, replace=False)
            v.reshape(-1, 4)[idx[:k], 0] = np.nan
            v.reshape(-1, 4)[idx[k:2 * k], 1] = np.inf
            v.reshape(-1, 4)[idx[2 * k:], 1] = -np.inf
        faces.append(v)
    return faces


# ------------------------------------------------------------------ views
def random_rotation(seed):
    """A rotation with roll, as a view matrix (no translation)."""
    q = np.random.default_rng(seed).standard_normal(4)
    q /= np.linalg.norm(q)
    return glam.from_scale_rotation_translation((1.0, 1.0, 1.0), q, (0.0, 0.0, 0.0))


def axis_view(face, handedness):
    direction, up = LOOK[face]
    look = glam.look_at_lh if handedness == LEFT else glam.look_at_rh
    return look(np.zeros(3, dtype=np.float32), np.array(direction, dtype=np.float32), np.array(up, dtype=np.float32))


# signed permutations of the axes (det +1) mapping the view's x and y to two world axes: the diagonal pixels of a square target
# tie |world a| == |world b| exactly
TIE_VIEWS = {
    "x_y": ((1, 0, 0), (0, 1, 0), (0, 0, 1)),      # view rows: looking along +Z, view x = X, view y = Y
    "x_z": ((1, 0, 0), (0, 0, -1), (0, 1, 0)),     # looking along +Y, view x = X, view y = -Z
    "y_z": ((0, 1, 0), (0, 0, 1), (1, 0, 0)),      # looking along +X, view x = Y, view y = Z
    "x_y_back": ((-1, 0, 0), (0, 1, 0), (0, 0, -1)),
}


def permutation_view(rows):
    m = np.eye(4, dtype=np.float32)
    m[:3, :3] = np.asarray(rows, dtype=np.float32).T     # storage m[c][r] = math[r][c]
    return m


def offaxis_projection(fov_deg, aspect, near=0.1, shift=(0.3, -0.2)):
    """A raw projection: the infinite reverse-Z perspective with its frustum sheared off the axis."""
    p = glam.perspective_infinite_reverse_lh(glam.to_radians(fov_deg), aspect, near).copy()
    p[2, 0], p[2, 1] = shift
    return p


# ------------------------------------------------------------------ frames
@dataclass
class SkyView:
    faces: list
    srgb: bool = False
    mips: str = "generated"
    view: np.ndarray = None
    projection: tuple = ("perspective", 60.0, 0.1)
    resolution: Tuple[int, int] = (64, 64)
    handedness: str = LEFT


def runner(backend, v: SkyView):
    r = TestRunner(backend, v.handedness)
    r.renderer.set_skybox(v.faces, srgb=v.srgb, mips=v.mips)
    r.renderer.set_camera_data(Camera(v.projection, glam.identity() if v.view is None else v.view))
    return r


def translucent_cube(r, view, alpha=0.5, colour=(0.25, 0.5, 0.75)):
    """An unlit blended cube 3 units in front of the camera: it covers the middle of the target and leaves the sky around it."""
    mat = r.renderer.add_material(PbrMaterial(albedo_value=(colour[0], colour[1], colour[2], alpha), unlit=True, transparency=BLEND))
    r.cube(mat, glam.mul(glam.inverse(view), glam.from_translation((0.0, 0.0, 3.0))))
    return np.array([colour[0], colour[1], colour[2], alpha], dtype=np.float32)


def draw(r, resolution, samples=1, frame_graph=None, upload=True, scissor_rows=None):
    r.renderer.set_aspect_ratio(resolution[0] / resolution[1])
    ev = r.renderer.evaluate()
    r.last_eval = ev
    r.base_rendergraph.add_to_graph(ev, resolution, samples, BaseRenderGraphSettings(clear_color=(0.0, 0.0, 0.0, 1.0)), frame_graph=frame_graph,
                                    upload=upload, scissor_rows=scissor_rows)
    return ev


def reference(r, resolution, desc=None, blob=None) -> "sref.Sky":
    """The float64 sky of the runner's last frame, from the uniform words the kernels read and the blob the frame uploaded."""
    ev = r.last_eval
    u = frame_uniforms(ev.camera, (0.0, 0.0, 0.0, 0.0), resolution)
    if desc is None:
        desc, blob = ev.skybox_desc, ev.skybox_texels
    return sref.reference_sky(u["inv_origin_view_proj"], resolution[0], resolution[1], desc, blob)


def render(backend, v: SkyView, samples=1) -> Tuple[TestRunner, "sref.Sky"]:
    r = runner(backend, v)
    draw(r, v.resolution, samples)
    return r, reference(r, v.resolution)
