"""A scene with three shadowed directional lights whose shadow indices differ from their handles, and a ten-step sequence of
DirectionalLightChanges (single fields, all four fields, empty masks, an index named twice, more than 64 entries in one call, the sun at
exactly -Y / +Y and back, distance 0 and back, negative / zero / NaN intensity), for tests/test_directional_light_updates.py."""
import numpy as np

from rend3_b200 import glam
from rend3_b200.world import LEFT, RIGHT, Camera, DirectionalLight, DirectionalLightChange, MeshBuilder, Object, PbrMaterial, Renderer

C = DirectionalLightChange
RES = (192, 108)
# handle -> resolution: the atlas places the 256 map first, so handle 1 is shadow index 0, handle 0 index 1, handle 2 index 2
LIGHTS = [DirectionalLight(color=(1.0, 1.0, 1.0), intensity=0.6, direction=(-1.0, -2.0, 0.5), distance=20.0, resolution=128),
          DirectionalLight(color=(0.4, 0.4, 0.6), intensity=0.4, direction=(0.5, -1.5, -1.0), distance=24.0, resolution=256),
          DirectionalLight(color=(0.9, 0.7, 0.5), intensity=0.3, direction=(0.2, -1.0, 0.9), distance=16.0, resolution=128)]


def many(n=70):
    """n entries cycling over the three lights, each one field: the last entries of each light and field decide the state."""
    out = []
    for k in range(n):
        t = 0.1 * k
        kind = k % 4
        change = (C(direction=(float(np.cos(t)), -1.5, float(np.sin(t)))) if kind == 0 else
                  C(intensity=0.25 + 0.005 * k) if kind == 1 else
                  C(color=(0.5 + 0.005 * k, 0.8, 1.0 - 0.004 * k)) if kind == 2 else
                  C(distance=18.0 + 0.05 * k))
        out.append((k % 3, change))
    return out


STEPS = [
    [],                                                                                           # 0: nothing (n = 0)
    [(0, C(color=(1.0, 0.6, 0.3))), (1, C(intensity=0.9)), (2, C(direction=(0.4, -1.0, 0.7)))],   # 1: single-field masks
    [(0, C(distance=31.0)), (1, C(direction=(-0.6, -1.3, -0.2))), (2, C(color=(0.2, 0.9, 0.4)))],  # 2: single-field masks
    [(0, C(color=(0.8, 0.8, 1.0), intensity=0.7, direction=(-0.3, -1.0, -0.6), distance=26.0)),     # 3: all four fields, an empty mask
     (1, C()),
     (2, C(color=(1.0, 0.9, 0.8), intensity=0.45, direction=(0.7, -1.1, 0.1), distance=19.0))],
    [(1, C(color=(1.0, 0.2, 0.2))), (1, C(intensity=0.5)), (1, C(color=(0.3, 0.6, 1.0), direction=(0.1, -1.0, 0.3))),   # 4: index named
     (0, C(distance=18.0)), (0, C(distance=24.0)), (2, C())],                                                              # twice, later wins
    many(),                                                                                       # 5: more than 64 entries in one call
    [(1, C(direction=(0.0, -1.0, 0.0))), (2, C(direction=(0.0, 1.0, 0.0))), (0, C(distance=0.0))],   # 6: sun at -Y / +Y, distance 0
    [(1, C(direction=(-0.5, -1.2, 0.3))), (2, C(direction=(0.3, -1.0, -0.4))), (0, C(distance=22.0)),  # 7: back; negative and zero
     (0, C(intensity=-0.4)), (2, C(intensity=0.0))],                                                   #    intensity
    [(1, C(intensity=float("nan")))],                                                             # 8: NaN intensity
    [(1, C(intensity=0.6)), (0, C(intensity=0.8)), (2, C(intensity=0.5, color=(0.6, 0.7, 0.9)))],   # 9: back
]
NAN_FRAMES = {8}   # the NaN intensity reaches every pixel the light shades


def world(left):
    """A ground plane and a field of cubes under the three lights."""
    from rend3_b200.runner import cube_mesh

    r = Renderer(LEFT if left else RIGHT, aspect_ratio=RES[0] / RES[1])
    lit = r.add_material(PbrMaterial(albedo_value=(0.6, 0.5, 0.4, 1.0), roughness_factor=0.6))
    plane = MeshBuilder.new([(-1, 0, -1), (-1, 0, 1), (1, 0, 1), (1, 0, -1)], LEFT).with_indices([0, 1, 2, 0, 2, 3] if left else [0, 2, 1, 0, 3, 2]).build()
    r.add_object(Object(r.add_mesh(plane), lit, glam.from_scale((10.0, 1.0, 10.0))))
    cube = r.add_mesh(cube_mesh())
    rng = np.random.default_rng(4)
    for _ in range(24):
        p = (float(rng.uniform(-6, 6)), 0.5, float(rng.uniform(-6, 6)))
        r.add_object(Object(cube, lit, glam.from_scale_rotation_translation((0.5, 0.5, 0.5), glam.QUAT_IDENTITY, p)))
    for light in LIGHTS:
        r.add_directional_light(light)
    return r


def camera(frame, left):
    eye = (0.5 + 0.05 * frame, 6.0 - 0.03 * frame, -10.0 + 0.06 * frame)
    return Camera(("perspective", 60.0, 0.1), (glam.look_at_lh if left else glam.look_at_rh)(eye, (0.0, 0.5, 0.0), (0.0, 1.0, 0.0)))


def same_bits(a, b):
    """Bit-identical arrays, any float32 NaN equal to any NaN (NaN payloads are not part of the rule)."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.names:   # field by field: a copy of a record array need not copy the padding between fields
        return all(same_bits(a[f], b[f]) for f in a.dtype.names)
    if a.dtype.itemsize % 4:
        return a.tobytes() == b.tobytes()
    x, y = a.view(np.uint32).ravel(), b.view(np.uint32).ravel()
    return bool(np.all((x == y) | (np.isnan(x.view(np.float32)) & np.isnan(y.view(np.float32)))))
