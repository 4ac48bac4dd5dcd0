"""Scenes where the shadow lookup is decided by ties, and the probe that reads the shadow factor back out of the HDR target.

A two-sided floor faces the viewer and the lights: either a pixel rectangle under the raw orthographic camera of
tests/shade_scenes.py (identity view), or a square on a slanted plane through the origin seen by a look-at camera (perspective or
orthographic, left- or right-handed), where the view, its inverse, the model-view and the perspective weights are all general.
Each light shines along the floor's normal, away from the viewer.  The
shadow passes cull front faces, so the floor's other winding writes the atlas: caster and receiver are the same plane at one
depth in the light's space, and every PCF compare sets a reference depth against a texel of that plane that is equal to it up to
rounding.  That is the "acne" regime of double-sided materials, foliage cards and thin walls, where a one-ulp difference in the
reference depth flips a tap.

The probe material has metallic 0, reflectance 0 and clear coat 0, so f0 = f90 = 0 and the specular term of surface_shading is
exactly 0 (opaque.wgsl:440-468); with roughness > 0, ambient 0 and albedo 1 a light's contribution is
(diffuse_pi * intensity) * (n.l * shadow).  Each light that carries colour does so in one channel of its own, so the channel
divided by the float64 value of the other factors recovers that light's shadow factor to a few float32 ulps.  Lights without
colour still take a lookup each (the kernels do not skip them), so the light count reaches the lights read from global memory
(past the 8 the shading kernels stage in shared memory).  The lights' resolutions are not powers of two, so neither is the
atlas, and the tiles sit away from the atlas origin.

Not built here: a translucent layer (blend_apply_kernel rounds every blended primitive to rgba16f, so the probe could read a
factor back only to about 2^-11, far too coarse for one-ulp flips; the kernel shades through the same shade_inputs and
shadow_pcf5), receivers with snz exactly 0 or 1, and footprints with u * W - 0.5 exactly an integer (both need view positions
placed to the ulp through R6 and light.view_proj, which these scenes do not construct)."""
from dataclasses import dataclass
from typing import Optional

import numpy as np

import raster_scenes
import shade_scenes
import shadow_lookup_reference as ref
from rend3_b200 import glam
from rend3_b200.layouts import CAMERA_VIEWPORT, DIRECTIONAL_LIGHT_DTYPE
from rend3_b200.routines import frame_uniforms
from rend3_b200.runner import TestRunner
from rend3_b200.world import CUTOUT, LEFT, OPAQUE, RIGHT, Camera, DirectionalLight, MeshBuilder, Object, PbrMaterial

F = np.float32
PI_F32 = F(3.14159265359)
CHANNEL = ((1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0))
AMBIENT = (0.0, 0.0, 0.0, 0.0)
# the slanted plane of the look-at scenes: its normal (towards the camera) and two unit vectors spanning it
PLANE_N = np.array([0.25, 1.0, -0.15]) / np.linalg.norm([0.25, 1.0, -0.15])
PLANE_T1 = np.cross(PLANE_N, [0.0, 0.0, 1.0]) / np.linalg.norm(np.cross(PLANE_N, [0.0, 0.0, 1.0]))
PLANE_T2 = np.cross(PLANE_N, PLANE_T1)


@dataclass
class Floor:
    """A two-sided probe floor: the pixel rectangle x0..x1, y0..y1 of a width x height target, on the plane
    z = z0 + slope_x * x + slope_y * y, lit by `n_lights` lights along the plane's normal whose shadow cameras are `distance`
    wide, optionally with the walkthrough's alpha checker (raster_scenes.cutout_texture) under the `sampler` filter.  With `eye`
    set, the floor is instead a square 8 units wide on the plane through the origin with normal PLANE_N, seen from `eye` by a
    look-at camera with `projection` in `handed` coordinates (rect, z0 and the slopes are then unused)."""
    width: int
    height: int
    rect: tuple
    n_lights: int
    distance: float = 240.0
    z0: float = 20.0
    slope_x: float = 0.0
    slope_y: float = 0.0
    sampler: Optional[str] = None
    eye: Optional[tuple] = None
    handed: str = LEFT
    projection: tuple = ("perspective", 60.0, 0.1)

    def normal(self):
        """The floor's normal towards the viewer; the lights shine along its negation."""
        if self.eye is not None:
            return tuple(float(c) for c in F(PLANE_N))
        return (self.slope_x, self.slope_y, -1.0)

    def material(self, texture=None):
        return PbrMaterial(albedo_value=(1.0, 1.0, 1.0, 1.0), roughness_factor=0.5, metallic_factor=0.0, reflectance=0.0, clearcoat_factor=0.0,
                           albedo_texture=texture, transparency=OPAQUE if texture is None else CUTOUT, alpha_cutout=0.5,
                           sample_type=self.sampler or "linear")

    def lights(self):
        """Resolutions 96 / 80 / 48, never a power of two.  The first, the one at index 8 (the first past the shared-memory stage)
        or else the last, and the last carry colour, one channel each."""
        carry = sorted({0, min(8, self.n_lights - 1), self.n_lights - 1})
        d = tuple(-c for c in self.normal())
        return [DirectionalLight(color=CHANNEL[carry.index(i)] if i in carry else (0.0, 0.0, 0.0), intensity=1.0, direction=d, distance=self.distance,
                                 resolution=(96, 80, 48)[i % 3]) for i in range(self.n_lights)]

    def triangles(self):
        """(4, 3, 3) positions: two triangles, then the same two reversed (shade_scenes' two-sided order).  For the pixel
        rectangle the first two face the camera."""
        if self.eye is not None:
            a, b, c, d = (F(4.0 * (sx * PLANE_T1 + sy * PLANE_T2)) for sx, sy in ((-1, -1), (1, -1), (1, 1), (-1, 1)))
            tris = np.array([[a, b, c], [a, c, d]], dtype=F)
            return np.concatenate([tris, tris[:, ::-1]])
        x0, y0, x1, y1 = self.rect
        tris = raster_scenes.oriented([((x0, y0), (x1, y0), (x1, y1)), ((x0, y0), (x1, y1), (x0, y1))])
        tris = np.concatenate([tris, tris[:, ::-1]])
        pos = np.zeros(tris.shape[:2] + (3,), dtype=F)
        pos[..., :2] = tris
        pos[..., 2] = F(self.z0) + F(self.slope_x) * pos[..., 0] + F(self.slope_y) * pos[..., 1]
        return pos


SCENES = {
    **{f"floor{n}": Floor(96, 64, (3, 2, 91, 61), n) for n in (1, 8, 9, 12)},
    # a narrower shadow camera: the floor runs past the right and lower edges of the tiles, so taps wrap at the atlas border
    # (Repeat) and fragments fall between the region test's bounds (1.5 texels in from the tile edge) and the edge itself
    "edges1": Floor(96, 64, (3, 2, 91, 61), 1, distance=100.0),
    "edges9": Floor(96, 64, (3, 2, 91, 61), 9, distance=100.0),
    # the walkthrough's checker: its holes cut the atlas too, and the kernels shade the floor through the textured path
    "cutout_nearest": Floor(96, 64, (3, 2, 91, 61), 1, sampler="nearest"),
    "cutout_linear": Floor(96, 64, (3, 2, 91, 61), 1, sampler="linear"),
    # a floor tilted against the view: the x, y and z terms of the shadow-space depth (lm * vp).z are all live
    "tilted9": Floor(96, 64, (3, 2, 91, 61), 9, slope_x=1.0 / 16.0, slope_y=-1.0 / 32.0),
    # power-of-two target and a 64 x 32 rectangle: the perspective weights, the view position, the normal and n.l = 1 are exact,
    # so the kernels' HDR is the oracle's bit for bit and a reordered tap sum shows
    "exact4": Floor(128, 64, (32, 16, 96, 48), 4),
    # look-at cameras: light.view_proj * inv_view, the model-view normal and (perspective) weights with w != 1 are all general
    **{f"perspective9_{h.lower()}": Floor(96, 64, None, 9, distance=40.0, eye=(1.0, 6.0, -7.0), handed=h) for h in (LEFT, RIGHT)},
    **{f"rotated_ortho1_{h.lower()}": Floor(96, 64, None, 1, distance=40.0, eye=(1.0, 6.0, -7.0), handed=h,
                                             projection=("orthographic", (12.0, 8.0, 40.0))) for h in (LEFT, RIGHT)},
}


def render(backend, name, samples, texture_table=False):
    """Draw scene `name` with shade_scenes' settings; `texture_table` binds a texture (the checker, used or not), so that the
    shading kernels take their TEX = true instantiation."""
    fl = SCENES[name]
    r = TestRunner(backend, fl.handed)
    tex = r.renderer.add_texture_2d(raster_scenes.cutout_texture()) if texture_table or fl.sampler else None
    mat = r.renderer.add_material(fl.material(tex if fl.sampler else None))
    pos = fl.triangles().reshape(-1, 3)
    mesh = MeshBuilder.new(pos, fl.handed).with_vertex_normals(np.tile(np.asarray(fl.normal(), dtype=F), (len(pos), 1)))
    if fl.sampler:
        mesh = mesh.with_vertex_texture_coordinates_0(pos[:, :2] / F(16.0))   # the checker repeats every 16 pixels
    r.renderer.add_object(Object(r.renderer.add_mesh(mesh.build()), mat, glam.identity()))
    for light in fl.lights():
        r.renderer.add_directional_light(light)
    if fl.eye is None:
        r.renderer.set_camera_data(Camera(("raw", glam.orthographic_lh(0.0, float(fl.width), float(fl.height), 0.0, 0.0, shade_scenes.DEPTH)),
                                          glam.identity()))
    else:
        r.renderer.set_aspect_ratio(fl.width / fl.height)
        look_at = glam.look_at_lh if fl.handed == LEFT else glam.look_at_rh
        r.renderer.set_camera_data(Camera(fl.projection, look_at(fl.eye, (0.0, 0.0, 0.0), (0.0, 1.0, 0.0))))
    shade_scenes.draw(r, shade_scenes.Scene(fl.width, fl.height, [], ambient=AMBIENT), samples)
    return r


def light_records(ev):
    n = int(np.frombuffer(ev.directional_buffer[:4], dtype=np.uint32)[0])
    return np.frombuffer(ev.directional_buffer[16:], dtype=DIRECTIONAL_LIGHT_DTYPE)[:n]


class Restated:
    """The float32 restatement of a rendered floor: per covered pixel (row-major over `mask`) the oracle's view position, each
    light's Lookup, n.l and the probe's HDR in the oracle's rounding.  `exact` marks the pixels whose centre lies more than 1e-3
    pixels inside one of the two drawn triangles (on an edge the raster's tie rule picks the record); `inside` (with `visible`
    given) is every pixel centre inside the floor."""

    def __init__(self, fl, ev, matrices, atlas, visible=None):
        mv, mvp = matrices[0]["model_view"], matrices[0]["model_view_proj"]
        self.identity_view = np.array_equal(mv, np.eye(4, dtype=F).reshape(16))
        tris = fl.triangles()
        clip = ref.mat_point(mvp, tris)                                             # (4, 3, 4)
        # framebuffer positions (y down) in float64, only to find the triangle that covers each pixel centre; the viewport draws
        # the winding whose framebuffer area is positive for left-handed cameras and negative for right-handed ones
        w = clip[..., 3].astype(np.float64)
        sx = (clip[..., 0] / w + 1.0) * fl.width * 0.5
        sy = (1.0 - clip[..., 1] / w) * fl.height * 0.5
        area = (sx[:, 1] - sx[:, 0]) * (sy[:, 2] - sy[:, 0]) - (sx[:, 2] - sx[:, 0]) * (sy[:, 1] - sy[:, 0])
        front = np.nonzero(area > 0 if fl.handed == LEFT else area < 0)[0]
        assert len(front) == 2, "the viewport should draw one winding of the floor"
        ys, xs = np.mgrid[0:fl.height, 0:fl.width]
        cx, cy = xs + 0.5, ys + 0.5
        owner = np.full(xs.shape, -1)
        margin = np.full(xs.shape, np.inf)
        for t in front:
            e = []
            for k in range(3):
                ax, ay, bx, by = sx[t, k], sy[t, k], sx[t, (k + 1) % 3], sy[t, (k + 1) % 3]
                e.append(np.sign(area[t]) * ((bx - ax) * (cy - ay) - (by - ay) * (cx - ax)) / np.hypot(bx - ax, by - ay))
            d = np.min(e, axis=0)                                                   # distance inside the triangle, in pixels
            owner = np.where(d > 0, t, owner)
            margin = np.where(d > 0, d, margin)
        self.mask = owner >= 0
        if visible is not None:
            self.inside = self.mask.copy()
            self.mask &= visible
        px, py, own = xs[self.mask], ys[self.mask], owner[self.mask]
        self.exact = margin[self.mask] > 1e-3            # away from the shared diagonal and the floor's edges
        self.vp, b = ref.view_position(px, py, fl.width, fl.height, clip[own], ref.mat_point(mv, tris)[own])
        u = frame_uniforms(ev.camera, AMBIENT, (fl.width, fl.height))
        self.lights = light_records(ev)
        self.lm = [ref.mat_mul(L["view_proj"], u["inv_view"]) for L in self.lights]
        self.lookups = [ref.lookup(self.vp, lm, L["atlas_offset"], L["atlas_size"], L["inv_resolution"], atlas) for lm, L in zip(self.lm, self.lights)]
        # vs_main's normal: normalize(mv3 * (inv_scale_sq * n)); fs_main normalises the interpolated normal again.  The view-space
        # light direction is normalize(view3 * -direction).  HDR = (inv_pi * colour) * (n.l * shadow)
        m = np.asarray(mv, dtype=F).reshape(4, 4)[:3, :3]                          # m[column] = column of the upper 3x3
        iss = F(1.0) / ref.dot3(m, m)
        sn = iss * np.asarray(fl.normal(), dtype=F)
        vn = ref.normalize3((m[0] * sn[0] + m[1] * sn[1]) + m[2] * sn[2])
        normal = ref.normalize3(ref.interpolate(b, np.broadcast_to(vn, (len(px), 3, 3))))
        view = np.asarray(u["view"], dtype=F).reshape(4, 4)[:3, :3]
        self.channel_light = []
        for c in range(3):
            carriers = [i for i, L in enumerate(self.lights) if L["color"][c] != 0]
            self.channel_light.append(carriers[0] if len(carriers) == 1 else None)
        self.nol = []
        for L in self.lights:
            nd = -np.asarray(L["direction"], dtype=F)
            lv = ref.normalize3((view[0] * nd[0] + view[1] * nd[1]) + view[2] * nd[2])
            self.nol.append(np.fmin(np.fmax(ref.dot3(normal, lv), F(0.0)), F(1.0)))
        inv_pi = F(1.0) / PI_F32
        self.hdr = np.zeros((len(self.vp), 3), dtype=F)
        for c, i in enumerate(self.channel_light):
            if i is not None:
                self.hdr[:, c] = (inv_pi * self.lights[i]["color"][c]) * (self.nol[i] * self.lookups[i].factor)

    def recover(self, hdr):
        """(N, 3) shadow factors of the channel-carrying lights from an HDR image (H, W, 4), in float64; NaN for a channel
        without a light."""
        h = np.asarray(hdr, dtype=np.float64)[self.mask][:, :3]
        out = np.full(h.shape, np.nan)
        for c, i in enumerate(self.channel_light):
            if i is not None:
                out[:, c] = h[:, c] / (float(F(1.0) / PI_F32) * float(self.lights[i]["color"][c]) * self.nol[i].astype(np.float64))
        return out

    def factors(self):
        """(N, 3) float32 factors of the channel-carrying lights, NaN where a channel carries none."""
        out = np.full((len(self.vp), 3), np.nan)
        for c, i in enumerate(self.channel_light):
            if i is not None:
                out[:, c] = self.lookups[i].factor
        return out


def restate(runner, name, atlas, visible=None):
    """The Restated frame of a runner that has drawn scene `name`, with `atlas` the atlas readback and `visible` (H, W) the pixels
    the floor covers (all of its rectangle when None)."""
    b = runner.backend
    return Restated(SCENES[name], runner.last_eval, b.readback_object_matrices(CAMERA_VIEWPORT, 0, len(runner.last_eval.object_buffer)), atlas, visible)


def wraps(o, atlas_shape):
    """(N,) sampled fragments with a tap whose bilinear footprint leaves the atlas, so that the Repeat wrap picks its texels."""
    h, w = atlas_shape
    out = np.zeros(len(o.flx), dtype=bool)
    for ix, iy in zip(o.ix, o.iy):
        out |= (ix < 0) | (ix + 1 >= w) | (iy < 0) | (iy + 1 >= h)
    return out & o.sampled


def in_bound_band(o, light):
    """(N,) fragments that the region test rejects with its bounds 1.5 texels in from the tile's far edges (factor 1) but would
    sample with bounds 0.5 texels in: flx and fly both past the 1.5 bound, one of them not past the 0.5 bound."""
    far = np.asarray(light["atlas_offset"], dtype=F) + np.asarray(light["atlas_size"], dtype=F)
    inv = np.asarray(light["inv_resolution"], dtype=F)
    b15, b05 = far - inv * F(1.5), far - inv * F(0.5)
    past = (o.flx > b15[0]) & (o.fly > b15[1])
    snz = o.sn[:, 2]
    return past & ((o.flx <= b05[0]) | (o.fly <= b05[1])) & (snz >= 0.0) & (snz <= 1.0)
