"""Scenes for the vertex-stage tests (tests/vertex_reference.py), aimed where a vertex stage goes wrong: perspective cameras of
both handednesses; objects with non-uniform scale and shear, so that inv_scale_sq changes the direction of smooth normals that
are not axis-aligned; vertex colours whose four bytes all differ; a floor whose triangles cross the near plane and reach past the
64w guard band; 4x silhouettes; normal maps of one texel value in every layout with explicit and generated tangents; and the
IEEE edges (a zero normal, an axis scaled by 0, a normal map without uv0).

`expected()` decides in float64 which primitive owns each pixel centre (1x) or sample (4x) and evaluates fs_main there.  A point
within MARGIN pixels of the boundary of a visible triangle's region (an edge or the near-plane line, as float64 edge functions
place it) is not decided: its pixel is left out, and so is a pixel where two objects overlap on screen."""
from dataclasses import dataclass, field, replace
from typing import List, Optional

import numpy as np

import raster_reference
import raster_scenes
import shade_reference as ref
import vertex_reference as vref
from rend3_b200 import glam
from rend3_b200.layouts import CAMERA_VIEWPORT, DIRECTIONAL_LIGHT_DTYPE, MAT_UNLIT
from rend3_b200.routines import BaseRenderGraphSettings
from rend3_b200.runner import TestRunner
from rend3_b200.world import BLEND, LEFT, RIGHT, Camera, CameraState, DirectionalLight, Mesh, Object, PbrMaterial, PointLight, Texture

MARGIN = 1.0 / 64.0            # pixels; R2 snaps vertices to 1/256 px
CLEAR = (0.1, 0.2, 0.3, 1.0)
AMBIENT = (0.03, 0.02, 0.05, 0.0)
GUARD = 64.0                   # R1: |x|, |y| <= 64 w


@dataclass
class Obj:
    pos: np.ndarray                         # (n, 3) f32
    normal: np.ndarray                      # (n, 3) f32
    indices: np.ndarray                     # (3m,) u32
    transform: np.ndarray                   # (4, 4) f32, [column][row]
    material: PbrMaterial
    colour: Optional[np.ndarray] = None     # (n, 4) u8
    tangent: Optional[np.ndarray] = None    # (n, 3) f32, the slot-2 attribute
    uv: Optional[np.ndarray] = None         # (n, 2) f32
    normal_map: Optional[tuple] = None      # RGBA8 bytes of a constant normal map (every mip level holds them)
    label: str = ""


@dataclass
class Scene:
    width: int
    height: int
    handedness: str
    view: np.ndarray
    objects: List[Obj]
    point_lights: List[PointLight] = field(default_factory=list)
    dir_lights: List[DirectionalLight] = field(default_factory=list)
    vfov: float = 60.0
    near: float = 0.5
    ambient: tuple = AMBIENT


# ------------------------------------------------------------------ meshes and transforms
def uv_sphere(n_lat, n_lon, winding):
    """A unit UV sphere with smooth outward normals (the positions), uv = (lon, lat) fractions; poles shared.  `winding` +1 or
    -1 picks the index order, so a handedness can see its outside."""
    lat = np.linspace(0.0, np.pi, n_lat + 1)[1:-1]
    lon = np.linspace(0.0, 2.0 * np.pi, n_lon, endpoint=False)
    ring = np.stack([np.outer(np.sin(lat), np.cos(lon)), np.repeat(np.cos(lat)[:, None], n_lon, 1), np.outer(np.sin(lat), np.sin(lon))], axis=-1)
    pos = np.concatenate([[[0.0, 1.0, 0.0]], ring.reshape(-1, 3), [[0.0, -1.0, 0.0]]])
    uv = np.concatenate([[[0.5, 0.0]], np.stack(np.meshgrid(lon / (2 * np.pi), (lat / np.pi)), -1).reshape(-1, 2), [[0.5, 1.0]]])
    idx = lambda i, j: 1 + i * n_lon + (j % n_lon)
    tris = []
    for j in range(n_lon):
        tris.append((0, idx(0, j + 1), idx(0, j)))
        tris.append((len(pos) - 1, idx(n_lat - 2, j), idx(n_lat - 2, j + 1)))
        for i in range(n_lat - 2):
            a, b, c, d = idx(i, j), idx(i, j + 1), idx(i + 1, j), idx(i + 1, j + 1)
            tris += [(a, b, d), (a, d, c)]
    t = np.array(tris, dtype=np.uint32)
    if winding < 0:
        t = t[:, [0, 2, 1]]
    pos32 = pos.astype(np.float32)
    return pos32, (pos32 / np.linalg.norm(pos32.astype(np.float64), axis=1, keepdims=True)).astype(np.float32), uv.astype(np.float32), t.reshape(-1)


def affine(rot_axis, angle, scale, shear, translation):
    """rotation(axis, angle) * shear * scale, then the translation, as f32 [column][row]: a shear puts a multiple of column 0 into
    column 1 and of column 1 into column 2, so the columns are not orthogonal."""
    a = np.asarray(rot_axis, dtype=np.float64) / np.linalg.norm(rot_axis)
    k = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    r = np.eye(3) + np.sin(angle) * k + (1 - np.cos(angle)) * k @ k
    sh = np.array([[1.0, shear, 0.0], [0.0, 1.0, shear], [0.0, 0.0, 1.0]])
    m = r @ sh @ np.diag(scale)
    out = np.eye(4)
    out[:3, :3] = m.T
    out[3, :3] = translation
    return out.astype(np.float32)


def colours(n, seed):
    """Per-vertex RGBA8 with four distinct bytes per vertex."""
    rng = np.random.default_rng(seed)
    return np.stack([rng.permutation(np.arange(16, 240, 3))[:4] for _ in range(n)]).astype(np.uint8)


def winding(handedness):
    return 1 if handedness == LEFT else -1


def sphere_obj(handedness, material, transform, seed, label, n_lat=10, n_lon=16, **kw):
    pos, nrm, uv, idx = uv_sphere(n_lat, n_lon, winding(handedness))
    return Obj(pos, nrm, idx, transform, material, colour=colours(len(pos), seed), label=label, **kw), uv


def floor_obj(handedness, forward, seed):
    """A quad at y = -1.5 from 4 units behind the camera to 40 in front, 3000 wide: its triangles cross the near plane and reach
    past the guard band.  Normals and colours vary per vertex, so the weights matter everywhere."""
    s = forward
    pos = np.array([[-1500, -1.5, -4 * s], [1500, -1.5, -4 * s], [1500, -1.5, 40 * s], [-1500, -1.5, 40 * s]], dtype=np.float32)
    nrm = np.array([[0.3, 1.0, 0.2], [-0.4, 1.0, 0.1], [0.2, 0.8, -0.5], [-0.1, 1.0, 0.6]])
    nrm = (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(np.float32)
    idx = np.array([0, 2, 1, 0, 3, 2], dtype=np.uint32)
    if handedness != LEFT:
        idx = idx.reshape(-1, 3)[:, [0, 2, 1]].reshape(-1)
    m = PbrMaterial(albedo_value=(0.9, 0.8, 0.7, 1.0), albedo_vertex="linear", roughness_factor=0.6, reflectance=0.5)
    return Obj(pos, nrm, idx, np.eye(4, dtype=np.float32), m, colour=colours(4, seed), label="floor")


def camera_view(handedness):
    eye = np.array([0.3, 0.2, 0.0])
    s = 1.0 if handedness == LEFT else -1.0
    centre = eye + np.array([0.05, -0.02, s])
    fn = glam.look_at_lh if handedness == LEFT else glam.look_at_rh
    return fn(eye.astype(np.float32), centre.astype(np.float32), np.array([0.0, 1.0, 0.0], dtype=np.float32)), s


def lights(forward, seed):
    rng = np.random.default_rng(seed + 500)
    pl = [PointLight(position=(float(rng.uniform(-6, 6)), float(rng.uniform(-1, 4)), float(forward * rng.uniform(4, 14))),
                     color=tuple(float(c) for c in rng.uniform(0.4, 1.0, 3)), radius=float(rng.uniform(12.0, 30.0)), intensity=float(rng.uniform(2.0, 6.0)))
          for _ in range(6)]
    dl = [DirectionalLight(color=(0.9, 0.8, 0.7), intensity=1.2, direction=(0.3, -0.8, 0.5 * forward), distance=1.0, resolution=32)]
    return pl, dl


# ------------------------------------------------------------------ scenes
def spheres_scene(handedness, seed=0):
    """Five spheres with rotation, non-uniform scale (0.25 - 4) and shear, lit and unlit, vertex albedo linear and sRGB, over the
    near-clipped floor."""
    view, s = camera_view(handedness)
    rng = np.random.default_rng(seed)
    objs = [floor_obj(handedness, s, seed + 1)]
    mats = [PbrMaterial(albedo_value=(0.8, 0.9, 0.7, 1.0), albedo_vertex="linear", roughness_factor=0.35, metallic_factor=0.2),
            PbrMaterial(albedo_value=(0.9, 0.7, 0.8, 1.0), albedo_vertex="srgb", roughness_factor=0.6, reflectance=0.8),
            PbrMaterial(albedo_value=(0.7, 0.8, 0.9, 0.9), albedo_vertex="linear", unlit=True),
            PbrMaterial(albedo_value=(1.0, 0.9, 0.8, 1.0), albedo_vertex="srgb", unlit=True),
            PbrMaterial(albedo_value=(0.6, 0.7, 0.8, 1.0), roughness_factor=0.2, metallic_factor=0.7, clearcoat_factor=0.3, clearcoat_roughness_factor=0.5)]
    scales = [(0.25, 1.0, 4.0), (1.6, 0.5, 0.9), (0.6, 1.3, 0.35), (1.0, 0.3, 1.0), (0.5, 1.5, 2.0)]
    places = [(-2.6, 1.7, 7.0), (0.0, 2.1, 8.0), (2.7, 1.6, 7.5), (-1.2, 4.0, 11.0), (1.8, 4.3, 11.0)]
    for k in range(5):
        axis = rng.normal(size=3)
        t = affine(axis, float(rng.uniform(0.5, 2.5)), np.array(scales[k]) * 0.9, 0.45 if k % 2 == 0 else 0.0,
                   np.array(places[k]) * np.array([1.0, 1.0, s]))
        o, _ = sphere_obj(handedness, mats[k], t, seed + 10 + k, f"sphere{k}")
        objs.append(o)
    pl, dl = lights(s, seed)
    return Scene(192, 128, handedness, view, objs, pl, dl)


NORMAL_LAYOUTS = {
    # name: (material fields, RGBA8 texel) - the swizzled texel's alpha differs from its red, so x from .w is visible
    "tricomponent": (dict(normal_kind="tricomponent"), (170, 100, 220, 255)),
    "bicomponent": (dict(normal_kind="bicomponent"), (90, 160, 0, 255)),
    "bicomponent_swizzled": (dict(normal_kind="bicomponent_swizzled"), (0, 170, 0, 80)),
    "tricomponent_ydown": (dict(normal_kind="tricomponent", normal_y_down=True), (150, 90, 230, 255)),
    "bicomponent_ydown": (dict(normal_kind="bicomponent", normal_y_down=True), (100, 180, 0, 255)),
}


def normal_map_scene(handedness, seed=0):
    """One sphere per normal-map layout with explicit tangents (varying, not orthogonal to the normal), and two with tangents
    from calculate_tangents; non-uniform scale and shear on all of them."""
    from rend3_b200.world import calculate_tangents
    view, s = camera_view(handedness)
    rng = np.random.default_rng(seed + 100)
    objs = []
    names = list(NORMAL_LAYOUTS) + ["tricomponent", "bicomponent_swizzled"]
    for k, name in enumerate(names):
        fields, texel = NORMAL_LAYOUTS[name]
        m = PbrMaterial(albedo_value=(0.8, 0.75, 0.7, 1.0), albedo_vertex="linear", roughness_factor=0.4, reflectance=0.6, **fields)
        x, y = -3.0 + 2.0 * (k % 4), 0.6 + 2.2 * (k // 4)
        t = affine(rng.normal(size=3), float(rng.uniform(0.5, 2.5)), np.array([0.7, 0.45, 1.4]) * rng.uniform(0.8, 1.1, 3), 0.4 if k % 2 else -0.3,
                   np.array([x, y, 9.0 * s]))
        o, uv = sphere_obj(handedness, m, t, seed + 20 + k, f"nmap_{name}" + ("_generated" if k >= len(NORMAL_LAYOUTS) else ""), normal_map=texel)
        o.uv = uv
        if k < len(NORMAL_LAYOUTS):
            tg = np.cross(o.normal.astype(np.float64), rng.normal(size=3)) + 0.5 * o.normal * rng.uniform(-1, 1, (len(o.pos), 1))
            tg += 0.3 * rng.normal(size=tg.shape)
            o.tangent = tg.astype(np.float32)
        else:
            o.tangent = calculate_tangents(o.pos, o.normal, o.uv, o.indices)
        objs.append(o)
    pl, dl = lights(s, seed)
    return Scene(192, 128, handedness, view, objs, pl, dl)


def ieee_scene(handedness=LEFT, seed=0):
    """A zero vertex normal on every vertex of one sphere, a sphere scaled by 0 along its local z (1 / 0 = inf, inf * 0 = NaN),
    and a normal-mapped sphere without uv0 (the tangent is absent: normalize(0) = NaN); next to an ordinary sphere."""
    view, s = camera_view(handedness)
    lit = PbrMaterial(albedo_value=(0.8, 0.7, 0.6, 1.0), albedo_vertex="linear", roughness_factor=0.5)
    objs = []
    o, _ = sphere_obj(handedness, lit, affine((1, 0, 0), 0.3, (0.9, 0.8, 1.1), 0.2, (-2.2, 1.8, 7.0 * s)), seed + 1, "zero_normal")
    o.normal = np.zeros_like(o.normal)
    objs.append(o)
    # local z scaled by 0 and the disc turned to face the camera: the flattened back half is culled
    o, _ = sphere_obj(handedness, lit, affine((0, 1, 0), 0.0, (1.0, 0.8, 0.0), 0.0, (0.4, 1.8, 7.0 * s)), seed + 2, "zero_scale")
    objs.append(o)
    fields, texel = NORMAL_LAYOUTS["tricomponent"]
    o, _ = sphere_obj(handedness, PbrMaterial(albedo_value=(0.7, 0.8, 0.6, 1.0), roughness_factor=0.4, **fields),
                      affine((0, 0, 1), 0.4, (0.8, 1.0, 0.9), 0.0, (2.8, 1.8, 7.0 * s)), seed + 3, "nmap_no_uv", normal_map=texel)
    objs.append(o)
    o, _ = sphere_obj(handedness, lit, affine((1, 1, 0), 0.7, (0.5, 1.0, 1.5), 0.3, (0.0, 4.2, 10.0 * s)), seed + 4, "ordinary")
    objs.append(o)
    pl, dl = lights(s, seed)
    return Scene(192, 128, handedness, view, objs, pl, dl)


SCENES = {
    "spheres_lh": lambda: spheres_scene(LEFT),
    "spheres_rh": lambda: spheres_scene(RIGHT, seed=1),
    "normal_maps_lh": lambda: normal_map_scene(LEFT),
    "normal_maps_rh": lambda: normal_map_scene(RIGHT, seed=1),
    "ieee": ieee_scene,
}


# ------------------------------------------------------------------ rendering
def mesh_of(o: Obj) -> Mesh:
    attrs = [(0, o.pos), (1, o.normal)]
    if o.tangent is not None:
        attrs.append((2, np.asarray(o.tangent, dtype=np.float32)))
    if o.uv is not None:
        attrs.append((3, o.uv))
    if o.colour is not None:
        attrs.append((5, o.colour))
    return Mesh(attrs, len(o.pos), np.asarray(o.indices, dtype=np.uint32))


def translucent_copy(o: Obj, alpha):
    """The object blended (transparency BLEND, albedo alpha `alpha`) and scaled by 1.08 about its centre: it encloses the opaque
    one, so its front faces lie over it and over the clear colour around the silhouette."""
    t = o.transform.astype(np.float64).copy()
    t[:3] *= 1.08
    m = replace(o.material, transparency=BLEND, albedo_value=tuple(list((o.material.albedo_value or (1, 1, 1, 1))[:3]) + [alpha]))
    return replace(o, transform=t.astype(np.float32), material=m, label=o.label + "_blend")


def all_objects(scene: Scene, translucent=None):
    objs = list(scene.objects)
    if translucent is not None:
        objs += [translucent_copy(o, translucent) for o in scene.objects if o.label.startswith("sphere")]
    return objs


def render(backend, scene: Scene, samples, texture_table=False, translucent=None):
    r = TestRunner(backend, scene.handedness)
    if texture_table:
        r.renderer.add_texture_2d(raster_scenes.cutout_texture())
    for o in all_objects(scene, translucent):
        m = o.material
        if o.normal_map is not None:
            tex = r.renderer.add_texture_2d(Texture(np.tile(np.array(o.normal_map, dtype=np.uint8), (8, 8, 1)), srgb=False, mips="generated"))
            m = replace(m, normal_texture=tex)
        r.renderer.add_object(Object(r.renderer.add_mesh(mesh_of(o)), r.renderer.add_material(m), o.transform))
    for l in scene.dir_lights:
        r.renderer.add_directional_light(l)
    for l in scene.point_lights:
        r.renderer.add_point_light(l)
    r.renderer.set_camera_data(Camera(("perspective", scene.vfov, scene.near), scene.view))
    r.renderer.set_aspect_ratio(scene.width / scene.height)
    ev = r.renderer.evaluate()
    r.last_eval = ev
    r.base_rendergraph.add_to_graph(ev, (scene.width, scene.height), samples, BaseRenderGraphSettings(ambient_color=scene.ambient, clear_color=CLEAR))
    return r


def material_record(o: Obj):
    """The material record as the kernels read it: a normal map's layout flags are only set when the material has one."""
    return (o.material if o.normal_map is None else replace(o.material, normal_texture=0)).to_record()


def needs_texture_table(scene: Scene):
    return any(o.normal_map is not None for o in scene.objects)


# ------------------------------------------------------------------ ownership
@dataclass
class Owners:
    """Per sample point (H, W, S): the owning object and triangle (-1 where no primitive covers it), whether the point is decided,
    and per object its triangle's flags."""
    obj: np.ndarray
    tri: np.ndarray
    decided: np.ndarray
    clipped: list           # per object, (T,) bool: a vertex with w < near or beyond the guard band
    sample_xy: np.ndarray   # (S, 2) sample offsets within the pixel


def _grad_px(c, width, height):
    """|grad| in pixels of the linear function c . (ndc_x, ndc_y, 1)."""
    return np.hypot(c[..., 0] * 2.0 / width, c[..., 1] * 2.0 / height)


def owners(scene: Scene, objs, mvp, samples, visible_sign, near):
    h, w = scene.height, scene.width
    offs = 0.5 + np.array(raster_reference.sample_offsets(samples), dtype=np.float64).reshape(-1, 2) / 256.0   # R7, 1/256 px from the centre
    ys, xs = np.mgrid[0:h, 0:w]
    fx = xs[..., None] + offs[:, 0]
    fy = ys[..., None] + offs[:, 1]
    nx, ny = vref.ndc(fx.ravel(), fy.ravel(), w, h)
    npts = nx.size
    best_w = np.full(npts, np.inf)
    own_o = np.full(npts, -1, dtype=np.int64)
    own_t = np.full(npts, -1, dtype=np.int64)
    undecided = np.zeros(npts, dtype=bool)
    clipped = []
    for oi, o in enumerate(objs):
        xyw, z = vref.clip_xyw(mvp[oi], o.pos.astype(np.float64))
        tris = np.asarray(o.indices, dtype=np.int64).reshape(-1, 3)
        clipped.append(np.array([bool(np.any(xyw[t, 2] < near) or np.any(np.abs(xyw[t, :2]) > GUARD * xyw[t, 2:3])) for t in tris]))
        for ti, t in enumerate(tris):
            p = xyw[t]
            det = np.linalg.det(p)
            if det == 0.0:
                continue
            sel = np.arange(npts)
            if np.all(p[:, 2] > 0):
                sx = (p[:, 0] / p[:, 2] + 1.0) * w * 0.5
                sy = (1.0 - p[:, 1] / p[:, 2]) * h * 0.5
                x0, x1, y0, y1 = sx.min() - 1, sx.max() + 1, sy.min() - 1, sy.max() + 1
                if x1 < 0 or y1 < 0 or x0 > w or y0 > h:
                    continue
                area = abs((sx[1] - sx[0]) * (sy[2] - sy[0]) - (sx[2] - sx[0]) * (sy[1] - sy[0]))
                sel = np.nonzero((fx.ravel() >= x0) & (fx.ravel() <= x1) & (fy.ravel() >= y0) & (fy.ravel() <= y1))[0]
            else:
                area = np.inf
            if len(sel) == 0:
                continue
            c = np.stack([np.cross(p[(i + 1) % 3], p[(i + 2) % 3]) for i in range(3)])
            g = p[:, 2] - z[t]                                      # w - z: the near plane of R1 (0 <= z <= w)
            cn = g @ c
            cs = np.concatenate([c, cn[None]])                      # three edges and the near-plane line
            q = np.stack([nx[sel], ny[sel], np.ones(len(sel))], axis=1)
            sd = np.sign(det) * (q @ cs.T) / _grad_px(cs, w, h)     # signed pixel distances, positive inside
            dmin = sd.min(axis=1)
            facing = np.sign(det) == visible_sign
            if not facing and area > 1.0:
                continue                                            # culled, and no snapping can flip its facing
            near_edge = np.abs(dmin) < MARGIN
            undecided[sel[near_edge]] = True
            if not facing:
                undecided[sel[dmin > -MARGIN]] = True              # a sliver whose snapped area might flip its facing
                continue
            inside = dmin >= MARGIN
            if not inside.any():
                continue
            pts = sel[inside]
            wi = det / np.sum(q[inside] @ c.T, axis=1)              # the clip w of the point: E_i = lambda_i det / w
            tie = np.isfinite(best_w[pts]) & (np.abs(wi - best_w[pts]) < 1e-3 * wi)
            undecided[pts[tie]] = True
            win = wi < best_w[pts]
            best_w[pts[win]] = wi[win]
            own_o[pts[win]] = oi
            own_t[pts[win]] = ti
    shape = (h, w, len(offs))
    return Owners(own_o.reshape(shape), own_t.reshape(shape), ~undecided.reshape(shape), clipped, offs)


# ------------------------------------------------------------------ expected values
@dataclass
class Expected:
    """Per pixel (H, W, 4) the float64 value the target holds, its sensitivity allowance and its f16 allowance, the pixels that are
    checked, and per-pixel census flags."""
    want: np.ndarray
    sens: np.ndarray
    f16: np.ndarray
    keep: np.ndarray
    single: np.ndarray           # (H, W) at most one object covers a sample
    covered: np.ndarray          # (H, W) every sample owned (depth > 0 after the min-resolve)
    empty: np.ndarray            # (H, W) no sample owned
    unlit: np.ndarray            # (H, W) every owned sample is an unlit material
    iss_moves: np.ndarray        # (H, W) setting inv_scale_sq := 1 moves the value beyond the bound
    clipped: np.ndarray          # (H, W) a sample's primitive was clipped by R1
    extrapolated: np.ndarray     # (H, W) a sample's primitive does not cover the pixel centre (4x)
    label: np.ndarray            # (H, W) object label of the first owned sample ("" where none)
    nan: np.ndarray              # (H, W) the fragment normal is NaN
    samples: int


def fragment_inputs(o: Obj, mv, mvp, tri_ids, fx, fy, width, height, iss=True, db=None):
    """(vp (m, 4), normal (m, 3), vcolor (m, 4), weights (m, 3), their f32 error bound (m, 3)) of object `o` for triangles
    `tri_ids` (m,) shaded at framebuffer points (fx, fy): vs_main per vertex, R6 weights (plus `db`, for the allowance), and the
    normal map's tangent basis where the object has one."""
    n = len(o.pos)
    vp_v, nrm_v, tan_v = vref.vs_main(mv, vref.attribute(o.pos, n, 3), vref.attribute(o.normal, n, 3), vref.attribute(o.tangent, n, 3), iss)
    col_v = vref.unpack_colour(o.colour, n)
    xyw, _ = vref.clip_xyw(mvp, vref.attribute(o.pos, n, 3))
    tris = np.asarray(o.indices, dtype=np.int64).reshape(-1, 3)[tri_ids]
    nx, ny = vref.ndc(fx, fy, width, height)
    b, eb = np.empty((len(tri_ids), 3)), np.empty((len(tri_ids), 3))
    for t in np.unique(tri_ids):
        k = tri_ids == t
        p = xyw[np.asarray(o.indices, dtype=np.int64).reshape(-1, 3)[t]]
        b[k], eb[k] = vref.weights(p, nx[k], ny[k]), vref.weight_error_bound(p, nx[k], ny[k])
    if db is not None:
        b = b + db
    lerp = lambda v: np.einsum("mi,mik->mk", b, v[tris])
    with np.errstate(all="ignore"):
        vp, normal, vcolor = lerp(vp_v), lerp(nrm_v), lerp(col_v)
        flags = int(material_record(o)["flags"])
        if o.normal_map is not None and not (flags & MAT_UNLIT):
            texel = np.broadcast_to(ref.f32(np.array(o.normal_map, dtype=np.float64) / 255.0), (len(tri_ids), 4))
            normal = vref.tbn_normal(normal, lerp(tan_v), vref.normal_map_value(texel, flags))
    return vp, normal, vcolor, b, eb


def light_inputs(scene: Scene, ev, view):
    """Point lights (view position, colour * intensity, radius) and directional lights (l, colour, lm = view_proj * inv_view)."""
    vm = vref.columns(view)
    pl_pos = np.array([np.concatenate([ref.f32(l.position), [1.0]]) @ vm for l in scene.point_lights]).reshape(-1, 4)[:, :3]
    pl_color = np.array([np.float32(l.color) * np.float32(l.intensity) for l in scene.point_lights], dtype=np.float64).reshape(-1, 3)
    pl_radius = np.array([l.radius for l in scene.point_lights], dtype=np.float32).astype(np.float64)
    n_dir = int(np.frombuffer(ev.directional_buffer[:4], dtype=np.uint32)[0])
    dl = np.frombuffer(ev.directional_buffer[16:], dtype=DIRECTIONAL_LIGHT_DTYPE)[:n_dir]
    d = -dl["direction"].astype(np.float64).reshape(-1, 3) @ vm[:3, :3]
    dir_l = d / np.linalg.norm(d, axis=1, keepdims=True)
    inv_view = vref.columns(CameraState(Camera(("perspective", scene.vfov, scene.near), view), scene.handedness, scene.width / scene.height).inv_view)
    lms = [(inv_view @ vref.columns(L["view_proj"])).reshape(16) for L in dl]
    return pl_pos, pl_color, pl_radius, dir_l, dl["color"].astype(np.float64).reshape(-1, 3), dl, lms


TIE = 1e-5


def shade(scene, o, mat_rec, vp, normal, vcolor, lights_in, atlas, sensitivity=True):
    """fs_main with the sensitivity allowance: (value, sens, shadow margin); only the value without `sensitivity`."""
    pl_pos, pl_color, pl_radius, dir_l, dir_color, dl, lms = lights_in
    mats = np.repeat(mat_rec[None], len(vp), axis=0)

    def shadows(v):
        if len(dl) == 0:
            return np.ones((len(v), 0)), np.full(len(v), np.inf)
        out = [ref.directional_shadow(v, lm, L["atlas_offset"], L["atlas_size"], L["inv_resolution"], atlas) for lm, L in zip(lms, dl)]
        return np.stack([x[0] for x in out], axis=1), np.min(np.stack([x[1] for x in out], axis=1), axis=1)

    def fn(v, nrm, pos, noh_scale):
        return ref.fs_main(v, nrm, mats, vcolor, scene.ambient, dir_l, dir_color, shadows(v)[0], pos, pl_color, pl_radius, noh_scale)
    if not sensitivity:
        return fn(vp[:, :3], normal, pl_pos, 1.0)
    want, sens = ref.with_sensitivity(vp[:, :3], normal, pl_pos, fn)
    return want, sens, shadows(vp[:, :3])[1]


def f16_step(v):
    return np.maximum(np.abs(v) * 2.0 ** -10, 2.0 ** -24)


def expected(scene: Scene, backend, runner, samples, atlas, objs=None, with_census=True) -> Expected:
    """The float64 reference for a frame rendered by `render` on `backend` (whose MV / MVP it reads back)."""
    objs = objs if objs is not None else scene.objects
    h, w = scene.height, scene.width
    recs = backend.readback_object_matrices(CAMERA_VIEWPORT, 0, len(objs))
    mvs, mvps = [r["model_view"] for r in recs], [r["model_view_proj"] for r in recs]
    visible_sign = -1.0 if scene.handedness == LEFT else 1.0      # R3 with PerCameraUniform.flags: Left culls det(xyw) > 0
    own = owners(scene, objs, mvps, samples, visible_sign, float(np.float32(scene.near)))
    lights_in = light_inputs(scene, runner.last_eval, scene.view)
    S = own.obj.shape[2]
    clear = np.float64(np.float32(CLEAR)) if samples == 1 else np.float16(CLEAR).astype(np.float64)
    val = np.broadcast_to(clear, (h, w, S, 4)).copy()
    sens = np.zeros((h, w, S, 4))
    ok = own.decided.copy()
    flags = {k: np.zeros((h, w, S), dtype=bool) for k in ("unlit", "iss", "clipped", "extra", "nan")}
    ys, xs = np.mgrid[0:h, 0:w]
    for oi, o in enumerate(objs):
        sel = own.obj == oi
        if not sel.any():
            continue
        py, px, si = np.nonzero(sel)
        tri = own.tri[sel]
        fx, fy = px + 0.5, py + 0.5
        vp, normal, vcolor, b, eb = fragment_inputs(o, mvs[oi], mvps[oi], tri, fx, fy, w, h)
        rec = material_record(o)
        v, sv, margin = shade(scene, o, rec, vp, normal, vcolor, lights_in, atlas)
        for i in range(3):                   # the f32 rounding of the weights, one weight at a time, either sign
            for sign in (-1.0, 1.0):
                db = np.zeros_like(eb)
                db[:, i] = sign * eb[:, i]
                vp2, n2, c2, _, _ = fragment_inputs(o, mvs[oi], mvps[oi], tri, fx, fy, w, h, db=db)
                v2 = shade(scene, o, rec, vp2, n2, c2, lights_in, atlas, sensitivity=False)
                sv = np.fmax(sv, np.abs(v2 - v))
        val[py, px, si], sens[py, px, si] = v, sv
        ok[py, px, si] &= margin > TIE
        flags["unlit"][py, px, si] = bool(rec["flags"] & MAT_UNLIT)
        flags["clipped"][py, px, si] = own.clipped[oi][tri]
        flags["extra"][py, px, si] = np.any(b < 0.0, axis=1)
        flags["nan"][py, px, si] = np.isnan(normal).any(axis=1)
        if with_census:
            vp1, n1, c1, _, _ = fragment_inputs(o, mvs[oi], mvps[oi], tri, fx, fy, w, h, iss=False)
            v1 = shade(scene, o, rec, vp1, n1, c1, lights_in, atlas, sensitivity=False)
            bound = ref.TOL * np.maximum(1.0, np.abs(v)) + sv + (f16_step(v) if samples == 4 else 0.0)
            flags["iss"][py, px, si] = np.any(np.abs(v1 - v) > bound, axis=1)
    owned = own.obj >= 0
    # one object per pixel: where two overlap on screen the pixel is left out (occlusion between objects is not what these scenes test)
    single = layers(scene, backend, objs, range(len(objs)), samples) <= 1
    keep = ok.all(axis=2) & single
    if samples == 1:
        want, s, f16 = val[:, :, 0], sens[:, :, 0], np.zeros((h, w, 4))
    else:
        want, s = val.mean(axis=2), sens.mean(axis=2)
        f16 = f16_step(val).mean(axis=2)                 # each sample rounds to rgba16f: half a step, or a whole one if it flips
    label = np.full((h, w), "", dtype=object)
    first = np.where(owned.any(axis=2), np.argmax(owned, axis=2), 0)
    oo = np.take_along_axis(own.obj, first[..., None], axis=2)[..., 0]
    for oi, o in enumerate(objs):
        label[(oo == oi) & owned.any(axis=2)] = o.label
    anyf = lambda k: (flags[k] & owned).any(axis=2)
    return Expected(want, s, f16, keep, single, owned.all(axis=2), ~owned.any(axis=2), (flags["unlit"] | ~owned).all(axis=2) & owned.any(axis=2),
                    anyf("iss"), anyf("clipped"), anyf("extra"), label, anyf("nan"), samples)


def layers(scene: Scene, backend, objs, which, samples=1):
    """Per pixel (H, W), how many of the objects `which` (indices into `objs`) cover a sample of it, counting undecided ones."""
    recs = backend.readback_object_matrices(CAMERA_VIEWPORT, 0, len(objs))
    sign = -1.0 if scene.handedness == LEFT else 1.0
    n = np.zeros((scene.height, scene.width), dtype=np.int64)
    for k in which:
        own = owners(scene, [objs[k]], [recs[k]["model_view_proj"]], samples, sign, float(np.float32(scene.near)))
        n += ((own.obj >= 0) | ~own.decided).any(axis=2)
    return n


def compare(got, e: Expected, mask=None, extra=0.0):
    """Channel values outside TOL + allowance (+ f16) of the reference on the kept pixels; NaN equals NaN.  Returns (bad (H, W, 4),
    number of values checked, fraction of them that needed more than TOL)."""
    got = np.asarray(got, dtype=np.float64)
    m = e.keep if mask is None else (e.keep & mask)
    m4 = np.broadcast_to(m[..., None], got.shape)
    base = ref.TOL * np.maximum(1.0, np.abs(e.want)) + e.f16 + extra
    err = np.abs(got - e.want)
    both_nan = np.isnan(got) & np.isnan(e.want)
    bad = m4 & ~both_nan & ~(np.nan_to_num(err, nan=np.inf) <= base + e.sens)
    n = int(np.count_nonzero(m4))
    needed = np.count_nonzero(m4 & ~both_nan & (np.nan_to_num(err, nan=np.inf) > base))
    return bad, n, (needed / n if n else 0.0)
