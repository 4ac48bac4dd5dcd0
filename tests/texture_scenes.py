"""Scenes for the textured-shading tests (tests/texture_reference.py), aimed where textureSampleGrad and get_pixel_data_inner go
wrong: camera-facing quads under the raw identity camera, so that every quad's texture coordinates and their derivatives are exact
dyadic numbers and a quad's footprint is exactly the number of texels per pixel it was built for (2^k: the fr == 0 return;
2^(k + 0.5) times 1 -+ 2e-2: the nearest sampler's tie, decided both ways; magnified; past the last level; anisotropic), plus a
perspective floor whose footprint sweeps through every level.  The textures are 64 x 16, 30 x 30 and 1 x 64 RGBA8 / RGBA8 sRGB
chains (width and height reach 1 at different levels), R8 and RG8 in slots that read their missing channels, BC1 with punch-through
alpha, BC5 snorm, BC7 and rgba16f beyond [0, 1]; the uv transforms mirror, rotate and shift by 2^20.  Materials: every AOMR layout
with and without its texture, every clear-coat layout, every normal layout with y up and down, vertex albedo linear and sRGB,
unlit, the nearest sampler, emissive and reflectance textures, a slot past the table; cutout quads whose alpha crosses the
threshold inside texels, whose uv transform makes the forward and the depth-pass decisions differ, and that cast into a shadow
map; a translucent textured quad over an opaque one.

`expected()` evaluates the reference at every decided sample point (tests/vertex_scenes.py's ownership) and returns the per-pixel
value, its bound and the census."""
from dataclasses import dataclass, field, replace
from typing import Dict

import numpy as np

import shade_reference as ref
import texture_reference as tref
import vertex_reference as vref
import vertex_scenes as vs
from rend3_b200 import glam
from rend3_b200.layouts import CAMERA_VIEWPORT, DIRECTIONAL_LIGHT_DTYPE, TEX_ALBEDO
from rend3_b200.routines import BaseRenderGraphSettings
from rend3_b200.runner import TestRunner
from rend3_b200.world import BLEND, CUTOUT, LEFT, Camera, DirectionalLight, Object, PbrMaterial, PointLight, Texture

W, H = 256, 128                 # 8 x 4 cells of 32 x 32 pixels
CELL = 32
CLEAR = vs.CLEAR
AMBIENT = (0.02, 0.03, 0.04, 0.0)
PAST_TABLE = 1000               # a texture handle past the table: its slot reads zeros


def _rng(seed):
    return np.random.default_rng(seed)


def textures():
    """name -> Texture; handles follow this order."""
    g = _rng(7)
    rgba = lambda h, w: g.integers(0, 256, (h, w, 4), dtype=np.uint8)
    normal = g.integers(70, 186, (16, 16, 4), dtype=np.uint8)
    bc1 = rgba(16, 16)
    bc1[..., 3] = np.where(g.random((16, 16)) < 0.3, 0, 255)            # punch-through texels
    alpha = np.zeros((8, 8, 4), dtype=np.uint8)
    alpha[..., :3] = rgba(8, 8)[..., :3]
    alpha[..., 3] = (np.arange(8)[None, :] * 34 + np.arange(8)[:, None] * 3).astype(np.uint8)   # crosses 0.4 inside texels
    alpha[3, 3, 3] = 102                                                 # exactly at the threshold 0.4
    return {
        "c64x16": Texture(rgba(16, 64)),
        "s30": Texture(rgba(30, 30), srgb=True),
        "t1x64": Texture(rgba(64, 1)),
        "r8": Texture(rgba(32, 32), channels=1),
        "rg8": Texture(rgba(32, 32), channels=2),
        "bc1": Texture(bc1, block_format="bc1"),
        "bc5s": Texture(rgba(16, 16), block_format="bc5s"),
        "bc7": Texture(rgba(16, 16), block_format="bc7"),
        "hdr": Texture(rgba(16, 16), storage="rgba16f"),
        "normal": Texture(normal),
        "alpha": Texture(alpha),
        "rgba": Texture(rgba(32, 32)),
    }


@dataclass
class Quad(vs.Obj):
    tex: Dict[str, str] = field(default_factory=dict)    # material slot field -> texture name (or PAST_TABLE)


@dataclass
class TexScene(vs.Scene):
    raw: bool = True
    tags: Dict[str, str] = field(default_factory=dict)   # label -> the edge it is there for


def uv_matrix(scale=(1.0, 1.0), angle=0.0, offset=(0.0, 0.0)):
    """uv_transform0 (columns) = translate(offset) * rotate(angle) * scale."""
    c, s = np.cos(angle), np.sin(angle)
    m = np.array([[c * scale[0], s * scale[0], 0.0], [-s * scale[1], c * scale[1], 0.0], [offset[0], offset[1], 1.0]])
    return m.astype(np.float32)


def quad(cell, material, uv_scale=(1.0, 1.0), z=0.5, label="", colour=None, size=CELL, depth=None, **tex):
    """A camera-facing quad on cell (column, row) of the raw camera's framebuffer: uv0 runs from (0, 0) at its top left to uv_scale at
    its bottom right, so the footprint is uv_scale * texture size / size texels per pixel.  With `depth` the quad lies at that view
    depth of the perspective camera of PERSPECTIVE instead, on the same cell."""
    cx, cy = cell
    x0, y0 = cx * CELL, cy * CELL
    nx = lambda px: px / (W / 2) - 1.0
    ny = lambda py: 1.0 - py / (H / 2)
    pos = np.array([[nx(x0), ny(y0 + size), z], [nx(x0), ny(y0), z], [nx(x0 + size), ny(y0), z], [nx(x0 + size), ny(y0 + size), z]], dtype=np.float32)
    su, sv = uv_scale
    uv = np.array([[0.0, sv], [0.0, 0.0], [su, 0.0], [su, sv]], dtype=np.float32)
    nrm = np.tile(np.array([[0.0, 0.0, -1.0]], dtype=np.float32), (4, 1))
    tan = np.tile(np.array([[1.0, 0.0, 0.0]], dtype=np.float32), (4, 1))
    idx = np.array([0, 1, 2, 0, 2, 3], dtype=np.uint32)
    if depth is not None:
        f = 1.0 / np.tan(np.radians(PERSPECTIVE[0]) / 2)
        pos = (pos.astype(np.float64) * [W / H * depth / f, depth / f, 0.0] + [0.0, 0.0, depth]).astype(np.float32)
    return Quad(pos, nrm, idx, np.eye(4, dtype=np.float32), material, colour=colour, tangent=tan, uv=uv, label=label, tex=tex)


PERSPECTIVE = (60.0, 0.5)       # vfov, near of the scenes that are not under the raw camera


def lit(**kw):
    base = dict(albedo_value=(0.9, 0.85, 0.8, 1.0), roughness_factor=0.55, metallic_factor=0.6, ao_factor=0.9, reflectance=0.7)
    base.update(kw)
    return PbrMaterial(**base)


def unlit_tex(**kw):
    return PbrMaterial(albedo_value=(1.0, 1.0, 1.0, 1.0), unlit=True, **kw)


def cells():
    return iter([(c, r) for r in range(4) for c in range(8)])


def levels_scene():
    """Unlit albedo-textured quads: the pixel is the sample itself."""
    at = cells()
    qs, tags = [], {}

    def add(label, tag, name, scale, **kw):
        qs.append(quad(next(at), unlit_tex(**{k: v for k, v in kw.items() if k != "colour"}), scale, label=label, colour=kw.get("colour"),
                       albedo_texture=name))
        tags[label] = tag
    # exact 2^k texels per pixel on the 64 x 16 chain: du/dx = s / 32, rho = 64 s / 32; v stays finer than u
    for k in range(4):
        add(f"pow2_{k}", "exact", "c64x16", (2.0 ** (k - 1), 2.0 ** (k - 1)))
    add("pow2_s30", "exact", "s30", (64.0 / 30.0, 32.0 / 30.0))          # 2 texels per pixel on 30 x 30: lambda exactly 1
    # the nearest tie 2^(k + 0.5) from both sides, and at the tie itself
    for k, sgn in ((1, -1), (1, 1), (2, -1), (2, 1), (0, 0)):
        s = 2.0 ** (k + 0.5 - 1) * (1.0 + sgn * 2e-2)
        add(f"tie_{k}_{'+' if sgn > 0 else '-' if sgn < 0 else '0'}", "tie", "c64x16", (s, s / 3.0), sample_type="nearest")
    add("magnified", "magnified", "c64x16", (0.1, 0.3))
    add("magnified_nearest", "magnified", "s30", (0.3, 0.2), sample_type="nearest")
    add("past_last", "past_last", "c64x16", (300.0, 90.0))
    add("past_last_1x64", "past_last", "t1x64", (3.0, 40.0))
    add("aniso", "aniso", "c64x16", (1.0, 1.0), uv_transform0=uv_matrix((4.0, 0.1)))
    add("mirror", "negative", "c64x16", (1.0, 1.0), uv_transform0=uv_matrix((-1.3, -0.7), offset=(0.21, -0.4)))
    add("rotated", "negative", "s30", (1.0, 1.0), uv_transform0=uv_matrix((1.5, 1.1), angle=0.52, offset=(-2.3, 0.7)))
    add("offset_2_20", "offset", "c64x16", (1.0, 1.0), uv_transform0=uv_matrix((0.75, 0.5), offset=(-2.0 ** 20, 2.0 ** 20)))
    add("npot", "npot", "s30", (1.4, 2.2))
    add("width1", "npot", "t1x64", (0.7, 1.9))
    add("srgb_bilinear", "srgb", "s30", (0.37, 0.41))
    add("r8_albedo", "missing", "r8", (1.3, 0.9))
    add("rg8_albedo", "missing", "rg8", (0.8, 1.2))
    add("bc1", "block", "bc1", (0.9, 1.3))
    add("bc1_small_levels", "block", "bc1", (3.0, 5.0))
    add("bc5s", "block", "bc5s", (1.1, 0.7))
    add("bc7", "block", "bc7", (2.3, 1.6))
    add("hdr", "hdr", "hdr", (1.2, 0.8))
    add("past_table", "past_table", PAST_TABLE, (1.0, 1.0))
    return TexScene(W, H, LEFT, glam.identity(), qs, tags=tags)


NORMAL_KINDS = ("tricomponent", "bicomponent", "bicomponent_swizzled")


def materials_scene():
    """Lit quads under point lights: one per AOMR layout with and without its texture, per clear-coat layout, per normal layout and
    y direction, vertex albedo linear and sRGB, unlit, nearest, emissive and reflectance textures, narrow textures in wide slots."""
    at = cells()
    qs, tags = [], {}
    colour = lambda seed: vs.colours(4, seed)

    def add(label, mat, scale=(0.9, 0.7), colour=None, **tex):
        qs.append(quad(next(at), mat, scale, label=label, colour=colour, **tex))
        tags[label] = label.split(":")[0]
    for kind in ("combined", "swizzled_split", "split", "bw_split"):
        extra = dict(metallic_texture="bc7", ao_texture="s30") if kind == "bw_split" else dict(ao_texture="s30") if kind == "split" else {}
        add(f"aomr:{kind}", lit(aomr_kind=kind), roughness_texture="rgba", **extra)
        add(f"aomr_absent:{kind}", lit(aomr_kind=kind))
    add("aomr_narrow:combined_rg8", lit(aomr_kind="combined"), roughness_texture="rg8")
    add("aomr_narrow:swizzled_r8", lit(aomr_kind="swizzled_split"), roughness_texture="r8")
    for kind in ("gltf_combined", "gltf_split", "bw_split"):
        add(f"clearcoat:{kind}", lit(clearcoat_kind=kind, clearcoat_factor=0.8, clearcoat_roughness_factor=0.9, roughness_factor=0.3),
            clearcoat_texture="c64x16", clearcoat_roughness_texture="rgba")
    for kind in NORMAL_KINDS:
        for down in (False, True):
            add(f"normal:{kind}{'_ydown' if down else ''}", lit(normal_kind=kind, normal_y_down=down), normal_texture="normal")
    add("vertex:linear", lit(albedo_vertex="linear"), colour=colour(3), albedo_texture="rgba")
    add("vertex:srgb", lit(albedo_vertex="srgb"), colour=colour(4), albedo_texture="s30")
    add("unlit", unlit_tex(albedo_vertex="srgb"), colour=colour(5), albedo_texture="rgba")
    add("nearest", lit(sample_type="nearest"), scale=(1.7, 2.9), albedo_texture="rgba", roughness_texture="c64x16", normal_texture="normal")
    add("emissive", lit(emissive=(2.0, 1.5, 3.0)), emissive_texture="hdr")
    add("emissive_ldr", lit(emissive=(0.7, 0.9, 1.1)), emissive_texture="rgba")
    add("reflectance", lit(metallic_factor=0.1), reflectance_texture="rgba")
    add("past_table", lit(), roughness_texture=PAST_TABLE, emissive_texture=PAST_TABLE)
    pl = [PointLight(position=(-0.6, 0.7, 0.1), color=(1.0, 0.9, 0.8), radius=6.0, intensity=3.0),
          PointLight(position=(0.8, -0.5, 0.2), color=(0.6, 0.8, 1.0), radius=5.0, intensity=2.0)]
    return TexScene(W, H, LEFT, glam.identity(), qs, point_lights=pl, ambient=AMBIENT, tags=tags)


def cutout_scene():
    """Unlit cutout quads (alpha_cutout 0.4) on the alpha texture, magnified so that the bilinear alpha crosses the threshold inside
    texels; some with a uv transform (the forward pass reads transformed coordinates, the depth pass the raw ones), one nearest, one
    with vertex alpha; a directional light shadows them into the atlas."""
    at = cells()
    qs, tags = [], {}

    def add(label, scale, colour=None, **kw):
        m = PbrMaterial(albedo_value=(1.0, 1.0, 1.0, 1.0), unlit=True, transparency=CUTOUT, alpha_cutout=0.4, **kw)
        q = quad(next(at), m, scale, label=label, colour=colour, depth=3.0, albedo_texture="alpha")
        q.indices = np.concatenate([q.indices, q.indices.reshape(-1, 3)[:, [0, 2, 1]].reshape(-1)])   # two-sided: the shadow camera sees the back
        qs.append(q)
        tags[label] = label
    add("plain", (1.0, 1.0))
    add("plain_fine", (0.45, 0.6))
    add("transformed", (1.0, 1.0), uv_transform0=uv_matrix((0.6, 1.3), angle=0.3, offset=(0.17, -0.2)))
    add("mirrored", (0.8, 0.9), uv_transform0=uv_matrix((-1.0, 1.0), offset=(0.05, 0.0)))
    add("nearest", (0.7, 0.8), sample_type="nearest")
    add("minified", (5.0, 3.0))
    add("vertex_alpha", (1.0, 1.0), colour=vs.colours(4, 9), albedo_vertex="linear")
    add("vertex_alpha_srgb", (0.9, 1.1), colour=vs.colours(4, 11), albedo_vertex="srgb")
    dl = [DirectionalLight(color=(1.0, 1.0, 1.0), intensity=1.0, direction=(0.3, -0.8, 0.5), distance=20.0, resolution=256)]
    return TexScene(W, H, LEFT, glam.identity(), qs, dir_lights=dl, vfov=PERSPECTIVE[0], near=PERSPECTIVE[1], raw=False, tags=tags)


def blend_scene():
    """A translucent textured quad (albedo alpha 0.55, texture alpha per texel) over an opaque textured one, and over the clear
    colour."""
    o = quad((1, 1), unlit_tex(), (1.3, 0.8), z=0.5, label="opaque", size=64, albedo_texture="s30")
    t = quad((2, 1), PbrMaterial(albedo_value=(1.0, 1.0, 1.0, 0.55), unlit=True, transparency=BLEND), (0.7, 1.1), z=0.6, label="blend",
             size=64, albedo_texture="rgba")
    return TexScene(W, H, LEFT, glam.identity(), [o, t], tags={"opaque": "opaque", "blend": "blend"})


def floor_scene():
    """A perspective floor in two halves, nearest and linear, on the 64 x 16 chain: the footprint grows with distance and is strongly
    anisotropic, so lambda sweeps through every level, through k + 0.5 and past the last level."""
    view = glam.look_at_lh(np.array([0.0, 1.0, 0.0], np.float32), np.array([0.0, 0.6, 4.0], np.float32), np.array([0.0, 1.0, 0.0], np.float32))
    qs = []
    for k, (x0, x1, st) in enumerate(((-8.0, 0.0, "nearest"), (0.0, 8.0, "linear"))):
        pos = np.array([[x0, 0.0, 0.5], [x0, 0.0, 60.0], [x1, 0.0, 60.0], [x1, 0.0, 0.5]], dtype=np.float32)
        uv = np.array([[0.0, 0.0], [0.0, 40.0], [3.0, 40.0], [3.0, 0.0]], dtype=np.float32) + np.float32(k * 0.37)
        nrm = np.tile(np.array([[0.0, 1.0, 0.0]], np.float32), (4, 1))
        qs.append(Quad(pos, nrm, np.array([0, 1, 2, 0, 2, 3], dtype=np.uint32), np.eye(4, dtype=np.float32), unlit_tex(sample_type=st),
                       uv=uv, label=f"floor_{st}", tex={"albedo_texture": "c64x16"}))
    return TexScene(W, H, LEFT, view, qs, raw=False, tags={q.label: "floor" for q in qs})


SCENES = {"levels": levels_scene, "materials": materials_scene, "cutout": cutout_scene, "blend": blend_scene, "floor": floor_scene}


# ------------------------------------------------------------------ rendering
def render(backend, scene: TexScene, samples):
    r = TestRunner(backend, scene.handedness)
    handles = {n: r.renderer.add_texture_2d(t) for n, t in textures().items()}
    for q in scene.objects:
        m = replace(q.material, **{k: (PAST_TABLE if v == PAST_TABLE else handles[v]) for k, v in q.tex.items()})
        r.renderer.add_object(Object(r.renderer.add_mesh(vs.mesh_of(q)), r.renderer.add_material(m), q.transform))
    for l in scene.dir_lights:
        r.renderer.add_directional_light(l)
    for l in scene.point_lights:
        r.renderer.add_point_light(l)
    cam = Camera(("raw", glam.identity()), scene.view) if scene.raw else Camera(("perspective", scene.vfov, scene.near), scene.view)
    r.renderer.set_camera_data(cam)
    r.renderer.set_aspect_ratio(scene.width / scene.height)
    ev = r.renderer.evaluate()
    r.last_eval = ev
    r.base_rendergraph.add_to_graph(ev, (scene.width, scene.height), samples, BaseRenderGraphSettings(ambient_color=scene.ambient, clear_color=CLEAR))
    return r


# ------------------------------------------------------------------ expected values
@dataclass
class Expected:
    want: np.ndarray        # (H, W, 4)
    bound: np.ndarray       # (H, W, 4): TOL + sensitivity + sampling bound (+ f16 at 4x)
    keep: np.ndarray        # (H, W) compared
    flagged: np.ndarray     # (H, W) left out: a nearest tie, a discard near its threshold, or a non-finite texel the error leaves open
    label: np.ndarray       # (H, W) object label ("" where none)
    discard: np.ndarray     # (H, W) the forward pass discards (decided pixels)
    census: dict            # name -> (H, W) bool


def _shade(scene, rec, px, bnd, vp, vnormal, vtangent, vcolor, pl):
    """fs_main on the pixel data, with the sensitivity allowance and the sampling bound carried through (each channel moved by its
    bound, either sign; the changes summed)."""
    pl_pos, pl_color, pl_radius = pl
    flags = int(rec["flags"])

    def run(p, v, nrm_in, pos, noh):
        nrm = tref.fragment_normal(p, flags, nrm_in, vtangent)
        return ref.fs_main(v, nrm, tref.untextured_records(p), np.ones((len(v), 4)), scene.ambient, (), (), None, pos, pl_color, pl_radius, noh)
    want, sens = ref.with_sensitivity(vp, vnormal, pl_pos, lambda v, n, p, noh: run(px, v, n, p, noh))
    extra = np.zeros_like(want)
    fields = list(tref.FIELDS) + ([("nmap", 4)] if px.nmap is not None else [])
    with np.errstate(all="ignore"):
        for name, nch in fields:
            for ch in range(nch):
                worst = np.zeros_like(want)
                for sign in (-1.0, 1.0):
                    worst = np.fmax(worst, np.abs(run(tref.perturbed(px, bnd, name, ch, sign), vp, vnormal, pl_pos, 1.0) - want))
                extra += worst
    return want, sens + extra


def point_lights_view(scene, view):
    vm = vref.columns(view)
    pos = np.array([np.concatenate([ref.f32(l.position), [1.0]]) @ vm for l in scene.point_lights]).reshape(-1, 4)[:, :3]
    col = np.array([np.float32(l.color) * np.float32(l.intensity) for l in scene.point_lights], dtype=np.float64).reshape(-1, 3)
    rad = np.array([l.radius for l in scene.point_lights], dtype=np.float32).astype(np.float64)
    return pos, col, rad


def expected(scene: TexScene, backend, runner, samples, which=None) -> Expected:
    """The reference frame of the objects `which` (indices, default all) as if no other object were drawn."""
    which = list(range(len(scene.objects))) if which is None else list(which)
    objs = [scene.objects[k] for k in which]
    h, w = scene.height, scene.width
    ev = runner.last_eval
    table = tref.Table(ev.texture_descs, ev.texture_texels)
    recs = backend.readback_object_matrices(CAMERA_VIEWPORT, 0, len(scene.objects))[which]
    mats = ev.material_buffer[which]       # the records the kernels read (set_materials): object k has material k
    mvs, mvps = [r["model_view"] for r in recs], [r["model_view_proj"] for r in recs]
    near = float(np.float32(scene.near)) if not scene.raw else 0.0
    own = vs.owners(scene, objs, mvps, samples, -1.0, near)
    S = own.obj.shape[2]
    clear = np.float64(np.float32(CLEAR)) if samples == 1 else np.float16(CLEAR).astype(np.float64)
    val = np.broadcast_to(clear, (h, w, S, 4)).copy()
    bnd = np.zeros((h, w, S, 4))
    flagged = np.zeros((h, w, S), dtype=bool)
    disc = np.zeros((h, w, S), dtype=bool)
    census = {k: np.zeros((h, w, S), dtype=bool) for k in ("fr0", "tie_lo", "tie_hi", "tie", "past_last", "magnified", "aniso", "negative",
                                                           "discard_near", "alt_differs")}
    pl = point_lights_view(scene, scene.view)
    for oi, o in enumerate(objs):
        rec = mats[oi]
        n = len(o.pos)
        vp_v, nrm_v, tan_v = vref.vs_main(mvs[oi], vref.attribute(o.pos, n, 3), vref.attribute(o.normal, n, 3), vref.attribute(o.tangent, n, 3))
        col_v = vref.unpack_colour(o.colour, n)
        xyw, _ = vref.clip_xyw(mvps[oi], vref.attribute(o.pos, n, 3))
        tris = np.asarray(o.indices, dtype=np.int64).reshape(-1, 3)
        uv_v = vref.attribute(o.uv, n, 2)
        for ti in range(len(tris)):
            sel = (own.obj == oi) & (own.tri == ti)
            if not sel.any():
                continue
            py, px_, si = np.nonzero(sel)
            t = tris[ti]
            fx, fy = px_ + 0.5, py + 0.5
            c = tref.coords(xyw[t], uv_v[t], fx, fy, w, h, tref.uv_transform(rec))
            nx, ny = vref.ndc(fx, fy, w, h)
            b = vref.weights(xyw[t], nx, ny)
            lerp = lambda a: b @ a[t]
            vcolor = lerp(col_v)
            pv, pb = tref.pixel_data(rec, c, vcolor, table)
            v, sb = _shade(scene, rec, pv, pb, lerp(vp_v)[:, :3], lerp(nrm_v), lerp(tan_v), vcolor, pl)
            d = tref.forward_discard(rec, c, vcolor, table) if rec["alpha_cutout"] > 0 else None
            fl = np.zeros(len(fx), dtype=bool)
            for s in pv.samples.values():
                fl |= s.tie | (s.nonfinite.any(-1) & s.moved)
                k = s.linear
                census["fr0"][py, px_, si] |= k & (s.lam > 0) & (s.fr == 0) & (s.level < len(table.levels(int(rec["textures"][TEX_ALBEDO])) or [0]) - 1)
                if not k:
                    frac = s.lam - np.floor(s.lam)
                    census["tie_lo"][py, px_, si] |= ~s.tie & (frac > 0.45) & (frac < 0.5)
                    census["tie_hi"][py, px_, si] |= ~s.tie & (frac > 0.5) & (frac < 0.55)
                    census["tie"][py, px_, si] |= s.tie
                    census["alt_differs"][py, px_, si] |= s.tie & (np.abs(s.alt - s.value) > s.bound()).any(-1)
                census["past_last"][py, px_, si] |= s.lam > len(table.levels(int(rec["textures"][TEX_ALBEDO])) or [0])
                census["magnified"][py, px_, si] |= s.lam < 0
                census["aniso"][py, px_, si] |= np.maximum(np.hypot(c.dudx, c.dvdx), np.hypot(c.dudy, c.dvdy)) > 8 * np.minimum(np.hypot(c.dudx, c.dvdx), np.hypot(c.dudy, c.dvdy))
                census["negative"][py, px_, si] |= (np.floor(c.u * 1e3) < 0) | (np.floor(c.v * 1e3) < 0)
            if d is not None:
                fl |= d.near
                census["discard_near"][py, px_, si] |= d.near
                disc[py, px_, si] = d.discard
                v = np.where(d.discard[:, None], clear, v)
                sb = np.where(d.discard[:, None], 0.0, sb)
            val[py, px_, si], bnd[py, px_, si], flagged[py, px_, si] = v, sb, fl
    owned = own.obj >= 0
    single = vs.layers(scene, backend, scene.objects, which, samples) <= 1
    ok = own.decided.all(axis=2) & single
    if samples == 1:
        want, b = val[:, :, 0], bnd[:, :, 0]
    else:
        want, b = val.mean(axis=2), bnd.mean(axis=2) + vs.f16_step(val).mean(axis=2)
    b = b + ref.TOL * np.maximum(1.0, np.abs(want))
    label = np.full((h, w), "", dtype=object)
    first = np.where(owned.any(axis=2), np.argmax(owned, axis=2), 0)
    oo = np.take_along_axis(own.obj, first[..., None], axis=2)[..., 0]
    for oi, o in enumerate(objs):
        label[(oo == oi) & owned.any(axis=2)] = o.label
    fl = flagged.any(axis=2)
    return Expected(want, b, ok & ~fl, ok & fl, label, (disc & owned).any(axis=2) & ok,
                    {k: (v & owned).any(axis=2) & ok & ~fl for k, v in census.items()} | {"flagged_tie": census["tie"].any(axis=2) & ok})


def compare(got, e: Expected, mask=None):
    """(bad (H, W, 4), number of values compared).  NaN equals NaN."""
    got = np.asarray(got, dtype=np.float64)
    m = e.keep if mask is None else (e.keep & mask)
    m4 = np.broadcast_to(m[..., None], got.shape)
    with np.errstate(invalid="ignore"):
        bad = m4 & ~(np.isnan(got) & np.isnan(e.want)) & ~(np.abs(got - e.want) <= e.bound)
    return bad, int(np.count_nonzero(m4))


# ------------------------------------------------------------------ the shadow pass
def shadow_decisions(scene: TexScene, backend, runner):
    """Per directional light, over its atlas region: (region slice, owner label (h, w), depth-pass discard, near flag, decided) of the
    cutout quads as the shadow camera sees them (depth.wgsl's predicate on raw coords0 with dpdy := dpdx)."""
    ev = runner.last_eval
    table = tref.Table(ev.texture_descs, ev.texture_texels)
    aw, ah = ev.shadow_target_size
    mats = ev.material_buffer
    n_dir = int(np.frombuffer(ev.directional_buffer[:4], dtype=np.uint32)[0])
    dl = np.frombuffer(ev.directional_buffer[16:], dtype=DIRECTIONAL_LIGHT_DTYPE)[:n_dir]
    out = []
    for L in dl:
        ox, oy = int(round(float(L["atlas_offset"][0]) * aw)), int(round(float(L["atlas_offset"][1]) * ah))
        vw, vh = int(round(float(L["atlas_size"][0]) * aw)), int(round(float(L["atlas_size"][1]) * ah))
        fake = replace(scene, width=vw, height=vh)
        mvps = [(vref.columns(o.transform) @ vref.columns(L["view_proj"])).astype(np.float32).reshape(16) for o in scene.objects]
        own = vs.owners(fake, scene.objects, mvps, 1, 1.0, 0.0)      # the light's view of the quads is their back
        disc, near = np.zeros((vh, vw), bool), np.zeros((vh, vw), bool)
        label = np.full((vh, vw), "", dtype=object)
        for oi, o in enumerate(scene.objects):
            n = len(o.pos)
            xyw, _ = vref.clip_xyw(mvps[oi], vref.attribute(o.pos, n, 3))
            tris = np.asarray(o.indices, dtype=np.int64).reshape(-1, 3)
            for ti, t in enumerate(tris):
                sel = (own.obj[..., 0] == oi) & (own.tri[..., 0] == ti)
                if not sel.any():
                    continue
                py, px_ = np.nonzero(sel)
                c = tref.coords(xyw[t], vref.attribute(o.uv, n, 2)[t], px_ + 0.5, py + 0.5, vw, vh, depth_pass=True)
                nx, ny = vref.ndc(px_ + 0.5, py + 0.5, vw, vh)
                valpha = vref.weights(xyw[t], nx, ny) @ vref.unpack_colour(o.colour, n)[t][:, 3]
                d = tref.depth_discard(mats[oi], c, valpha, table)
                disc[py, px_], near[py, px_], label[py, px_] = d.discard, d.near, o.label
        out.append(((slice(oy, oy + vh), slice(ox, ox + vw)), label, disc, near, own.decided[..., 0]))
    return out
