"""A world whose materials change from frame to frame, for r3_update_materials / r3_update_materials_device.

`MaterialWorld` is a world.Renderer with textured cubes: opaque, cutout and blend materials, textured and untextured, two shadowed
directional lights and three point lights.  Its materials change only through `Renderer.update_material`, so each frame's expected
state is `Renderer.evaluate()`: the full material table (what r3_set_materials uploads) and the stale indices (what the update calls
scatter).  `script` lists the edits of each frame; every material keeps its transparency, so the objects' sort info never changes."""
from __future__ import annotations

from dataclasses import replace

import numpy as np

from rend3_b200.scenes import cube_example_camera, random_unit_quaternions, subdivided_cube_mesh, trs_matrices
from rend3_b200.world import BLEND, CUTOUT, LEFT, DirectionalLight, Object, PbrMaterial, PointLight, Renderer, Texture

f32 = np.float32

# material handles of MaterialWorld
OPAQUE_TEX, OPAQUE_VALUE, CUTOUT_TEX, CUTOUT_VALUE, BLEND_VALUE, BLEND_TEX, EMISSIVE = range(7)


class MaterialWorld:
    """`discard=False` leaves out the cutout material whose alpha comes from a texture, so that no material discards per fragment;
    `blend=False` puts no object on a blend material (the materials stay in the table)."""

    def __init__(self, n_objects: int = 400, seed: int = 11, resolution=(256, 160), discard: bool = True, blend: bool = True):
        self.rng = rng = np.random.default_rng(seed)
        r = self.r = Renderer(LEFT, aspect_ratio=resolution[0] / resolution[1])
        meshes = [r.add_mesh(subdivided_cube_mesh(k, with_uv=True)) for k in (1, 2)]
        img = rng.integers(0, 256, (32, 32, 4), dtype=np.uint8)
        alpha = rng.integers(0, 256, (16, 16, 4), dtype=np.uint8)
        self.textures = [r.add_texture_2d(Texture(img, srgb=True)), r.add_texture_2d(Texture(alpha, srgb=True))]
        t0, t1 = self.textures
        for m in (PbrMaterial(albedo_texture=t0, roughness_factor=0.5),
                  PbrMaterial(albedo_value=(0.7, 0.6, 0.5, 1.0), roughness_factor=0.8),
                  PbrMaterial(albedo_texture=t1, roughness_factor=0.6, transparency=CUTOUT, alpha_cutout=0.5),
                  PbrMaterial(albedo_value=(0.4, 0.8, 0.4, 0.8), roughness_factor=0.7, transparency=CUTOUT, alpha_cutout=0.5),
                  PbrMaterial(albedo_value=(0.3, 0.6, 0.9, 0.5), roughness_factor=0.4, transparency=BLEND),
                  PbrMaterial(albedo_texture=t0, albedo_value=(1.0, 1.0, 1.0, 0.6), roughness_factor=0.3, transparency=BLEND),
                  PbrMaterial(albedo_value=(0.2, 0.2, 0.2, 1.0), emissive=(0.5, 0.1, 0.0), roughness_factor=0.9)):
            r.add_material(m)
        r.set_camera_data(cube_example_camera(8.0))
        for d in ((-1.0, -4.0, 2.0), (2.0, -3.0, -1.0)):
            r.add_directional_light(DirectionalLight(color=(1, 1, 1), intensity=0.6, direction=d, distance=80.0, resolution=256))
        for _ in range(3):
            r.add_point_light(PointLight(position=tuple(rng.uniform(-12, 12, 3)), color=tuple(rng.uniform(0.3, 1.0, 3)), radius=15.0, intensity=3.0))
        used = [OPAQUE_TEX, OPAQUE_VALUE, CUTOUT_VALUE, EMISSIVE] + ([CUTOUT_TEX] if discard else []) + ([BLEND_VALUE, BLEND_TEX] if blend else [])
        if not discard:
            r.update_material(CUTOUT_TEX, replace(r.materials[CUTOUT_TEX], albedo_texture=None, albedo_value=(0.9, 0.9, 0.9, 1.0)))
        transforms = trs_matrices(rng.uniform(-14.0, 14.0, (n_objects, 3)).astype(f32), random_unit_quaternions(rng, n_objects),
                                  rng.uniform(0.5, 1.4, (n_objects, 1)).astype(f32))
        for i in range(n_objects):
            r.add_object(Object(meshes[i % 2], used[int(rng.integers(0, len(used)))], transforms[i]))
        self.discard = discard

    def edit(self, handle: int, **changes):
        self.r.update_material(handle, replace(self.r.materials[handle], **changes))

    def uv_scroll(self, du: float, dv: float, scale: float = 1.0):
        return np.array([[scale, 0.0, 0.0], [0.0, scale, 0.0], [du, dv, 1.0]], dtype=f32)   # columns of a Mat3


def script(w: MaterialWorld):
    """The edits of frames 0 .. 6, applied to `w` one frame at a time (a generator: evaluate between the steps).  Frame 6 edits every
    material (the dense form).  Without `w.discard`, no edit makes a material discard per fragment."""
    t0, t1 = w.textures
    past = len(w.textures) + 5                                              # a texture slot past the table reads 0
    yield "albedo, emissive, roughness 0, metallic"
    w.edit(OPAQUE_VALUE, albedo_value=(0.2, 0.5, 0.9, 1.0), metallic_factor=0.7)
    w.edit(EMISSIVE, emissive=(0.0, 2.0, 0.5))
    w.edit(OPAQUE_TEX, roughness_factor=0.0)
    yield "uv_transform0"
    w.edit(OPAQUE_TEX, uv_transform0=w.uv_scroll(0.25, 0.1), roughness_factor=0.5)
    w.edit(CUTOUT_TEX, uv_transform0=w.uv_scroll(0.5, -0.3, 2.0))
    w.edit(BLEND_TEX, uv_transform0=w.uv_scroll(0.1, 0.1, 0.5))
    yield "texture slots, one past the table"
    w.edit(OPAQUE_TEX, albedo_texture=past)
    w.edit(OPAQUE_VALUE, albedo_texture=t1)
    w.edit(EMISSIVE, albedo_texture=t0)
    yield "ALBEDO_ACTIVE off"
    w.edit(CUTOUT_TEX, albedo_texture=None, albedo_value=None)
    w.edit(CUTOUT_VALUE, albedo_value=None)
    w.edit(OPAQUE_TEX, albedo_texture=t0)
    yield "ALBEDO_ACTIVE on, another alpha_cutout"
    if w.discard:
        w.edit(CUTOUT_TEX, albedo_texture=t0, alpha_cutout=0.3)
    else:
        w.edit(CUTOUT_TEX, albedo_value=(0.6, 0.3, 0.3, 0.7), alpha_cutout=0.3)
    w.edit(CUTOUT_VALUE, albedo_value=(0.4, 0.8, 0.4, 0.8))
    yield "alpha_cutout past the albedo alpha"
    w.edit(CUTOUT_VALUE, alpha_cutout=0.9)
    w.edit(CUTOUT_TEX, alpha_cutout=0.7)
    w.edit(BLEND_VALUE, albedo_value=(0.9, 0.2, 0.2, 0.3))
    yield "every material"
    for h in range(len(w.r.materials)):
        w.edit(h, roughness_factor=float(w.rng.uniform(0.1, 0.9)), emissive=tuple(w.rng.uniform(0.0, 0.3, 3)))
    yield "end"


def frames(w: MaterialWorld):
    """(label, EvalOutput) per frame: the edits of `script` applied, then Renderer.evaluate."""
    steps = script(w)
    label = next(steps)
    for nxt in steps:
        yield label, w.r.evaluate()
        label = nxt


def updates(ev):
    """(indices or None, records) of the frame's stale materials: None (the dense form) when every material is stale."""
    stale = ev.material_stale
    if len(stale) == len(ev.material_buffer):
        return None, ev.material_buffer.copy()
    return stale.copy(), ev.material_buffer[stale.astype(np.int64)]
