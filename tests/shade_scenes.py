"""Scenes for the shading tests whose fragment inputs are known in closed form.

Pixel-aligned quads, one object each with its own material, normal and vertex colour, seen through the raw orthographic camera
of tests/raster_scenes.py (identity view) with a deeper range, glam.orthographic_lh(0, W, H, 0, 0, DEPTH).  A pixel centre inside a
quad at depth z has the view position (px + 0.5, py + 0.5, z) in real arithmetic, and every vertex carries the same normal and
colour, so tests/shade_reference.py can evaluate fs_main there without re-running the vertex stage.  Quad edges lie on integer
pixels, so with four samples every sample of a pixel belongs to one quad and the resolve is the one shaded value in half precision.
The directional lights of the material grid get a shadow camera DIR_DISTANCE wide around the origin, which holds no geometry, so
their shadow factor is exactly 1; shadow_scene casts real shadows, and the reference takes its factors from the atlas readback."""
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

import raster_scenes
from rend3_b200 import glam
from rend3_b200.routines import BaseRenderGraphSettings
from rend3_b200.runner import TestRunner
from rend3_b200.world import BLEND, LEFT, Camera, DirectionalLight, MeshBuilder, Object, PbrMaterial, PointLight

DEPTH = 64.0
DIR_DISTANCE = 1.0
CLEAR = (0.1, 0.2, 0.3, 1.0)
AMBIENT = (0.03, 0.02, 0.05, 0.0)


@dataclass
class Quad:
    x0: int
    y0: int
    x1: int
    y1: int
    z: float
    material: PbrMaterial
    normal: tuple = (0.0, 0.0, -1.0)
    vcolor: tuple = (255, 255, 255, 255)
    two_sided: bool = False     # both windings: drawn by the shadow passes whichever way the light faces it


@dataclass
class Scene:
    width: int
    height: int
    quads: List[Quad]
    point_lights: List[PointLight] = field(default_factory=list)
    dir_lights: List[DirectionalLight] = field(default_factory=list)
    ambient: tuple = AMBIENT
    depth: float = DEPTH


# ------------------------------------------------------------------ rendering
def _quad_mesh(q: Quad):
    tris = raster_scenes.oriented([((q.x0, q.y0), (q.x1, q.y0), (q.x1, q.y1)), ((q.x0, q.y0), (q.x1, q.y1), (q.x0, q.y1))])
    if q.two_sided:
        tris = np.concatenate([tris, tris[:, ::-1]])
    n = 3 * len(tris)
    pos = np.zeros((n, 3), dtype=np.float32)
    pos[:, :2] = tris.reshape(-1, 2)
    pos[:, 2] = q.z
    return (MeshBuilder.new(pos, LEFT).with_vertex_normals(np.tile(np.asarray(q.normal, dtype=np.float32), (n, 1)))
            .with_vertex_color_0(np.tile(np.asarray(q.vcolor, dtype=np.uint8), (n, 1))).build())


def build(backend, scene: Scene, texture_table=False, translucent=None):
    """A TestRunner with the scene's quads, lights and camera.  `texture_table` binds a texture no material uses, so the shading
    kernels take their TEX = true instantiation; `translucent` (an alpha) adds a blended copy of every quad in front."""
    r = TestRunner(backend, LEFT)
    if texture_table:
        r.renderer.add_texture_2d(raster_scenes.cutout_texture())
    for q in scene.quads:
        mat = r.renderer.add_material(q.material)
        r.renderer.add_object(Object(r.renderer.add_mesh(_quad_mesh(q)), mat, glam.identity()))
    if translucent is not None:
        for front in translucent_copy(scene, translucent).quads:
            r.renderer.add_object(Object(r.renderer.add_mesh(_quad_mesh(front)), r.renderer.add_material(front.material), glam.identity()))
    for l in scene.dir_lights:
        r.renderer.add_directional_light(l)
    for l in scene.point_lights:
        r.renderer.add_point_light(l)
    r.renderer.set_camera_data(Camera(("raw", glam.orthographic_lh(0.0, float(scene.width), float(scene.height), 0.0, 0.0, scene.depth)),
                                      glam.identity()))
    return r


def translucent_copy(scene: Scene, alpha):
    """The scene's quads one unit nearer, blended (transparency BLEND) with albedo alpha `alpha`."""
    quads = []
    for q in scene.quads:
        m = PbrMaterial(**{**q.material.__dict__, "transparency": BLEND})
        a = m.albedo_value or (1.0, 1.0, 1.0, 1.0)
        m.albedo_value = (a[0], a[1], a[2], alpha)
        quads.append(Quad(q.x0, q.y0, q.x1, q.y1, q.z + 1.0, m, q.normal, q.vcolor))
    return Scene(scene.width, scene.height, quads, scene.point_lights, scene.dir_lights, scene.ambient, scene.depth)


def draw(r, scene: Scene, samples, scissor_rows=None):
    ev = r.renderer.evaluate()
    r.last_eval = ev
    r.base_rendergraph.add_to_graph(ev, (scene.width, scene.height), samples,
                                    BaseRenderGraphSettings(ambient_color=scene.ambient, clear_color=CLEAR), scissor_rows=scissor_rows)


def render(backend, scene: Scene, samples, **kw):
    scissor_rows = kw.pop("scissor_rows", None)
    r = build(backend, scene, **kw)
    draw(r, scene, samples, scissor_rows)
    return r


# ------------------------------------------------------------------ closed-form fragment inputs
@dataclass
class Fragments:
    """The covered pixels of a scene and what fs_main receives there, in float64 (view space = world space)."""
    mask: np.ndarray       # (H, W) covered
    owner: np.ndarray      # (H, W) quad index, -1 where uncovered
    vp: np.ndarray         # (N, 3) for the covered pixels in row-major order
    normal: np.ndarray
    vcolor: np.ndarray
    mat: np.ndarray        # (N,) MATERIAL_DTYPE


def fragments(scene: Scene) -> Fragments:
    owner = np.full((scene.height, scene.width), -1, dtype=np.int64)
    for k, q in enumerate(scene.quads):     # quads do not overlap
        owner[max(q.y0, 0):q.y1, max(q.x0, 0):q.x1] = k
    mask = owner >= 0
    ys, xs = np.nonzero(mask)
    o = owner[mask]
    z = np.array([np.float32(q.z) for q in scene.quads], dtype=np.float64)
    vp = np.stack([xs + 0.5, ys + 0.5, z[o]], axis=1)
    normal = np.array([q.normal for q in scene.quads], dtype=np.float32).astype(np.float64)[o]
    vcolor = np.array([q.vcolor for q in scene.quads], dtype=np.float64)[o] / 255.0
    recs = np.stack([q.material.to_record() for q in scene.quads])
    return Fragments(mask, owner, vp, normal, vcolor, recs[o])


def light_arrays(scene: Scene):
    """The point-light records as fs_main reads them (view space = world space), colours times intensity."""
    pl_pos = np.array([l.position for l in scene.point_lights], dtype=np.float32).reshape(-1, 3).astype(np.float64)
    pl_color = np.array([np.float32(l.color) * np.float32(l.intensity) for l in scene.point_lights], dtype=np.float64).reshape(-1, 3)
    pl_radius = np.array([l.radius for l in scene.point_lights], dtype=np.float32).astype(np.float64)
    return pl_pos, pl_color, pl_radius


@dataclass
class Expected:
    """The float64 fs_main of a rendered scene at its covered pixels (N, 4), the sensitivity allowance, and per pixel (N,) the
    smallest decision margin of any directional light's shadow lookup and the shadow factors (N, D)."""
    f: Fragments
    want: np.ndarray
    sens: np.ndarray
    shadow_margin: np.ndarray
    shadow: np.ndarray
    sampled: np.ndarray

    def image(self, values, fill=0.0):
        img = np.full(self.f.mask.shape + values.shape[1:], fill, dtype=np.float64)
        img[self.f.mask] = values
        return img


def expected(scene: Scene, ev, atlas) -> Expected:
    """The reference for a frame rendered with `ev` (the runner's last evaluation): directional lights in the order of its light
    buffer, each with its shadow factor from `atlas` (the shadow atlas readback, identical on every path)."""
    import shade_reference as ref
    from rend3_b200.layouts import DIRECTIONAL_LIGHT_DTYPE
    f = fragments(scene)
    n_dir = int(np.frombuffer(ev.directional_buffer[:4], dtype=np.uint32)[0])
    dl = np.frombuffer(ev.directional_buffer[16:], dtype=DIRECTIONAL_LIGHT_DTYPE)[:n_dir]
    d = dl["direction"].astype(np.float64).reshape(-1, 3)
    dir_l = -d / np.linalg.norm(d, axis=1, keepdims=True)
    dir_color = dl["color"].astype(np.float64).reshape(-1, 3)
    pl_pos, pl_color, pl_radius = light_arrays(scene)

    def shadows(vp):
        if n_dir == 0:
            return np.ones((len(vp), 0)), np.full((len(vp), 0), np.inf), np.zeros((len(vp), 0), dtype=bool)
        out = [ref.directional_shadow(vp, L["view_proj"], L["atlas_offset"], L["atlas_size"], L["inv_resolution"], atlas) for L in dl]
        return [np.stack([o[k] for o in out], axis=1).reshape(len(vp), n_dir) for k in range(3)]

    def fn(vp, normal, pos, noh_scale):
        return ref.fs_main(vp, normal, f.mat, f.vcolor, scene.ambient, dir_l, dir_color, shadows(vp)[0], pos, pl_color, pl_radius, noh_scale)
    want, sens = ref.with_sensitivity(f.vp, f.normal, pl_pos, fn)
    factor, margin, sampled = shadows(f.vp)
    return Expected(f, want, sens, margin.min(axis=1, initial=np.inf), factor, sampled)


def light_evaluations(scene: Scene, delta=0.0):
    """forward_light_evaluations() of a single-sample frame if every fragment-light distance d were compared with r + delta: per
    lit fragment, every directional light, and each point light with d < r + delta (every one for a roughness-0 fragment, and
    every one whose radius is not positive)."""
    import shade_reference as ref
    f = fragments(scene)
    px = ref.Pixel(f.mat, f.vcolor, f.normal)
    pl_pos, _, pl_radius = light_arrays(scene)
    lit = ~px.unlit
    count = np.full(len(f.vp), len(scene.dir_lights), dtype=np.int64)
    for p, r in zip(pl_pos, pl_radius):
        d = np.sqrt(np.sum((p - f.vp) ** 2, axis=1))
        with np.errstate(all="ignore"):
            count += ~(r > 0) | (d < r + delta) | (px.roughness == 0.0)
    return int(np.sum(count[lit]))


def light_evaluation_bounds(scene: Scene):
    """The range forward_light_evaluations() may take when the view position is off by up to 8 f32 ulps of its largest
    coordinate (the perspective weights round): (low, high), equal when no fragment lies that close to a radius."""
    u = 8.0 * 2.0 ** -24 * float(np.abs(fragments(scene).vp).max())
    return light_evaluations(scene, -u), light_evaluations(scene, u)


def untie_radii(scene: Scene, rel=1e-4):
    """Grow each positive point-light radius by steps of 3 rel until no fragment centre lies within `rel` of it (relative), so
    that f32 rounding of the view position cannot decide whether d^2 < r^2.  Returns the scene."""
    f = fragments(scene)
    for l in scene.point_lights:
        if not l.radius > 0 or not np.isfinite(l.radius):
            continue
        d = np.sqrt(np.sum((np.float32(l.position).astype(np.float64) - f.vp) ** 2, axis=1))
        while np.min(np.abs(d / np.float64(np.float32(l.radius)) - 1.0)) <= rel:
            l.radius = float(np.float32(l.radius * (1.0 + 3.0 * rel)))
    return scene


# ------------------------------------------------------------------ scenes
GRID_W, GRID_H = 130, 53   # neither a multiple of the 32 x 8 shading tile; the last tile column and row hold no quad


def _unit(rng, n, z_max=-0.2):
    v = rng.normal(size=(n, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    v[:, 2] = np.minimum(v[:, 2], z_max)      # mostly facing the viewer
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def material_grid(seed=0, roughness=None):
    """12 x 7 cells of 8 x 6 pixels at pixel (2 + 8i, 1 + 6j), each its own material and normal.  Sweeps perceptual roughness
    0.05 - 1, metallic 0 / 0.5 / 1, reflectance 0 / 0.5 / 1, clear coat with the clear-coat roughness above and below the base,
    AO < 1, emissive, unlit, and vertex albedo linear and sRGB."""
    rng = np.random.default_rng(seed)
    rough = [0.05, 0.1, 0.2, 0.35, 0.5, 0.75, 1.0]
    quads = []
    normals = _unit(rng, 84)
    for k in range(84):
        i, j = k % 12, k // 12
        m = PbrMaterial(albedo_value=tuple(float(v) for v in np.append(rng.uniform(0.2, 1.0, 3), 1.0)),
                        roughness_factor=rough[k % 7] if roughness is None else roughness, metallic_factor=[0.0, 0.5, 1.0][(k // 7) % 3],
                        reflectance=[0.0, 0.5, 1.0][(k // 3) % 3])
        kind = k % 12
        if kind == 1:
            m.clearcoat_factor, m.clearcoat_roughness_factor = 0.6, 0.9      # above the base roughness: the remap raises it
        elif kind == 2:
            m.clearcoat_factor, m.clearcoat_roughness_factor = 0.6, 0.01     # below: max() keeps the base
        elif kind == 3:
            m.ao_factor = 0.35
        elif kind == 4:
            m.emissive = (0.2, 0.1, 0.05)
        elif kind == 5 and roughness is None:
            m.unlit = True
        elif kind == 6:
            m.albedo_vertex = "linear"
        elif kind == 7:
            m.albedo_vertex = "srgb"
        vcolor = tuple(int(v) for v in rng.integers(0, 256, 4))
        z = float(rng.integers(32, 160)) / 8.0
        quads.append(Quad(2 + 8 * i, 1 + 6 * j, 10 + 8 * i, 7 + 6 * j, z, m, tuple(normals[k]), vcolor))
    return Scene(GRID_W, GRID_H, quads)


def random_point_lights(n, seed=0, width=GRID_W, height=GRID_H, radius=(8.0, 40.0)):
    rng = np.random.default_rng(seed + 1000)
    return [PointLight(position=(float(rng.uniform(-10, width + 10)), float(rng.uniform(-10, height + 10)), float(rng.uniform(-4.0, 24.0))),
                       color=tuple(float(c) for c in rng.uniform(0.2, 1.0, 3)), radius=float(rng.uniform(*radius)), intensity=float(rng.uniform(1.0, 4.0)))
            for _ in range(n)]


def dir_lights(n, seed=0):
    rng = np.random.default_rng(seed + 2000)
    out = []
    for _ in range(n):
        d = rng.normal(size=3)
        d[2] = abs(d[2]) + 0.3
        out.append(DirectionalLight(color=tuple(float(c) for c in rng.uniform(0.2, 1.0, 3)), intensity=float(rng.uniform(0.5, 2.0)),
                                    direction=tuple(float(c) for c in d / np.linalg.norm(d)), distance=DIR_DISTANCE, resolution=32))
    return out


def grid_with_lights(n_point, n_dir=1, seed=0, **kw):
    s = material_grid(seed, **kw)
    s.point_lights = random_point_lights(n_point, seed)
    s.dir_lights = dir_lights(n_dir, seed)
    return s


TANGENT_FACTORS = (1.0 - 1e-6, 1.0, 1.0 + 1e-6, 1.0 + 5e-4, 1.0 + 2e-3)


def tangent_layout(factor, seed=0):
    """One quad covering whole 32 x 8 tiles of a 160 x 40 target at z = 10, and lights tangent to tile boxes at factor x radius
    from the nearest fragment centre: off a face (along x), off an edge (x and y) and off a corner (x, y and z)."""
    rng = np.random.default_rng(seed)
    m = PbrMaterial(albedo_value=(0.8, 0.7, 0.6, 1.0), roughness_factor=0.6, reflectance=0.5)
    quads = [Quad(0, 0, 160, 40, 10.0, m, (0.3, -0.2, -0.93))]
    lights = []
    for k, (tx, ty) in enumerate([(1, 1), (2, 2), (3, 3), (1, 3), (3, 1)]):
        r = float(rng.uniform(3.0, 9.0))
        x_hi, y_hi = 32.0 * tx + 31.5, 8.0 * ty + 7.5          # the last fragment centres of tile (tx, ty)
        dist = r * factor
        kind = k % 3
        if kind == 0:
            pos = (x_hi + dist, 8.0 * ty + 4.0, 10.0)
        elif kind == 1:
            pos = (x_hi + dist / np.sqrt(2.0), y_hi + dist / np.sqrt(2.0), 10.0)
        else:
            pos = (x_hi + dist / np.sqrt(3.0), y_hi + dist / np.sqrt(3.0), 10.0 - dist / np.sqrt(3.0))
        lights.append(PointLight(position=tuple(float(np.float32(p)) for p in pos), color=(1.0, 0.9, 0.8), radius=r, intensity=3.0))
    return Scene(160, 40, quads, lights, dir_lights(1, seed))


def pythagorean_layout():
    """Lights at integer offsets (3k, 4k) from pixel centres in the same z plane with radius 5k: fragments at exactly d = r."""
    m = PbrMaterial(albedo_value=(0.6, 0.8, 0.7, 1.0), roughness_factor=0.4, reflectance=0.5)
    quads = [Quad(0, 0, 96, 24, 6.0, m, (0.0, 0.0, -1.0))]
    lights = [PointLight(position=(10.5 + 3 * k + 20 * k, 6.5 + 4 * k, 6.0), color=(1.0, 1.0, 1.0), radius=5.0 * k, intensity=2.0) for k in (1, 2, 3)]
    return Scene(96, 24, quads, lights, [])


def far_layout():
    """View coordinates near 1e4 (z) with radii near 1e-2: a light lights one or two fragments."""
    m = PbrMaterial(albedo_value=(0.9, 0.9, 0.9, 1.0), roughness_factor=0.5, reflectance=0.5)
    z = 10000.0
    quads = [Quad(0, 0, 64, 16, z, m, (0.0, 0.0, -1.0))]
    # each light 0.005 from one fragment centre with a radius of 0.012 - 0.022: f32 steps at 1e4 are 0.001, so the count is exact
    lights = [PointLight(position=(4.5 + 9 * k + 0.004, 8.5, z - 0.003), color=(1.0, 1.0, 1.0), radius=0.012 + 0.002 * k, intensity=5.0)
              for k in range(6)]
    return Scene(64, 16, quads, lights, [], depth=2.0 * z)


def half_covered_layout(seed=0):
    """Quads that cover the left half of some tiles, every other tile row, and leave whole tiles empty, in a 100 x 45 target."""
    rng = np.random.default_rng(seed)
    quads = []
    for ty in range(0, 6, 2):
        for tx in range(4):
            if (tx + ty) % 3 == 2:
                continue
            m = PbrMaterial(albedo_value=(0.7, 0.5, 0.4, 1.0), roughness_factor=float(rng.uniform(0.1, 1.0)), metallic_factor=0.5)
            quads.append(Quad(32 * tx, 8 * ty, min(32 * tx + 16, 100), min(8 * ty + 8, 45), float(rng.integers(16, 100)) / 8.0, m,
                              tuple(_unit(rng, 1)[0])))
    return Scene(100, 45, quads, random_point_lights(40, seed, 100, 45, radius=(3.0, 15.0)), dir_lights(1, seed))


DEGENERATE_RADII = {"zero": 0.0, "negative": -12.0, "nan": float("nan"), "inf": float("inf"), "huge": 1e20, "tiny": 1e-23}


SHADOW_W, SHADOW_H = 128, 64


def shadow_scene(n_dir, seed=0, distance=100.0):
    """A floor of four quads lit by `n_dir` directional lights that shine from +z (direction.z < 0), so the shadow passes cull the
    floor (front faces) and leave its texels clear, and two-sided 8 x 8 occluders 4 - 20 units above it, which write the only
    depths.  Each light's 128-texel map covers `distance` around the origin: the far part of the floor fails the any() region
    test or lies outside 0 <= z <= 1, where the factor is exactly 1."""
    rng = np.random.default_rng(seed + 3000)
    quads = []
    for k, (x0, y0, x1, y1) in enumerate([(0, 0, 64, 32), (64, 0, 128, 32), (0, 32, 64, 64), (64, 32, 128, 64)]):
        m = PbrMaterial(albedo_value=(0.9, 0.8, 0.7, 1.0), roughness_factor=[0.3, 0.6, 0.9, 0.45][k], metallic_factor=[0.0, 0.5, 0.0, 1.0][k])
        quads.append(Quad(x0, y0, x1, y1, [4.0, 6.0, 5.0, 3.0][k], m, (0.1, -0.05, 0.99)))
    occ = PbrMaterial(albedo_value=(0.4, 0.5, 0.6, 1.0), roughness_factor=0.5)
    for j in range(3):
        for i in range(6):
            x, y = 6 + 20 * i + int(rng.integers(0, 4)), 4 + 20 * j + int(rng.integers(0, 4))
            quads.append(Quad(x, y, x + 8, y + 8, float(rng.integers(10, 26)), occ, (0.0, 0.0, 1.0), two_sided=True))
    lights = []
    for _ in range(n_dir):
        d = np.array([rng.uniform(-0.5, 0.5), rng.uniform(-0.5, 0.5), -rng.uniform(0.7, 1.0)])
        lights.append(DirectionalLight(color=tuple(float(c) for c in rng.uniform(0.3, 1.0, 3)), intensity=float(rng.uniform(0.5, 1.5)),
                                       direction=tuple(float(c) for c in d / np.linalg.norm(d)), distance=distance, resolution=128))
    return Scene(SHADOW_W, SHADOW_H, quads, random_point_lights(4, seed, SHADOW_W, SHADOW_H), lights)


def degenerate_light_scene(kind, seed=0):
    """The material grid under ordinary lights plus one degenerate record: a radius from DEGENERATE_RADII, colour 0, or a light
    exactly on a fragment's view position."""
    s = untie_radii(grid_with_lights(6, 1, seed))
    if kind in DEGENERATE_RADII:
        s.point_lights.append(PointLight(position=(60.0, 25.0, 4.0), color=(0.9, 0.8, 0.7), radius=DEGENERATE_RADII[kind], intensity=2.0))
    elif kind == "colour0":
        s.point_lights.append(PointLight(position=(60.0, 25.0, 4.0), color=(0.0, 0.0, 0.0), radius=30.0, intensity=2.0))
    elif kind == "at_fragment":
        q = s.quads[30]
        s.point_lights.append(PointLight(position=(q.x0 + 2.5, q.y0 + 1.5, float(np.float32(q.z))), color=(1.0, 1.0, 1.0), radius=10.0, intensity=2.0))
    else:
        raise ValueError(kind)
    return s


DEGENERATE_KINDS = list(DEGENERATE_RADII) + ["colour0", "at_fragment"]
