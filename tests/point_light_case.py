"""Seeded PointLightManager sequences (add, update, remove with holes, an all-dead table, growth past the size, and NaN / inf / negative /
zero radius and intensity) applied alike to world.py's Renderer and to a backend's handle table, and the small walkthrough scene of
tests/test_point_lights.py."""
import numpy as np

from rend3_b200.layouts import POINT_LIGHT_SOURCE_DTYPE
from rend3_b200.world import PointLight

f32 = np.float32
SPECIAL = [0.0, -0.0, -1.5, np.nan, np.inf, -np.inf]


def random_light(rng, special=True):
    pos = rng.normal(size=3) * 10.0
    col = rng.random(3)
    radius = float(rng.uniform(0.5, 20.0))
    intensity = float(rng.uniform(0.0, 5.0))
    if special and rng.random() < 0.3:
        radius = float(rng.choice(SPECIAL))
    if special and rng.random() < 0.3:
        intensity = float(rng.choice(SPECIAL))
    if special and rng.random() < 0.1:
        pos[rng.integers(0, 3)] = rng.choice([np.nan, np.inf, -np.inf])
    if special and rng.random() < 0.1:
        col[rng.integers(0, 3)] = rng.choice([np.nan, np.inf, 0.0])
    return PointLight(position=tuple(float(v) for v in pos), color=tuple(float(v) for v in col), radius=radius, intensity=intensity)


def records(lights):
    """POINT_LIGHT_SOURCE_DTYPE records of PointLights (None: a zero record)."""
    out = np.zeros(len(lights), dtype=POINT_LIGHT_SOURCE_DTYPE)
    for i, l in enumerate(lights):
        if l is not None:
            out[i] = (l.position, l.color, l.radius, l.intensity)
    return out


def sequence(seed, steps=12):
    """A list of steps; a step is a list of (handle, PointLight or None = remove), each handle named once per step."""
    rng = np.random.default_rng(seed)
    size, out = 0, []
    for step in range(steps):
        kind = rng.integers(0, 5) if step else 0
        if step == steps // 2:   # every handle removed: an all-dead table
            ops = [(h, None) for h in range(size)]
        elif kind == 0 or size == 0:   # adds, some past the end (growth with dead handles between)
            n = int(rng.integers(1, 40))
            base = size + int(rng.integers(0, 6))
            ops = [(base + k, random_light(rng)) for k in range(n)]
        else:   # a mix of updates, removals (holes) and adds beyond the size
            hs = rng.permutation(size + 8)[: int(rng.integers(1, size + 8))]
            ops = [(int(h), None if rng.random() < 0.35 else random_light(rng)) for h in hs]
        out.append(ops)
        size = max([size] + [h + 1 for h, _ in ops])
    return out


def apply_to_world(renderer, ops):
    for h, l in ops:
        if l is None:
            renderer.remove_point_light(h)
        else:
            renderer.update_point_light(h, l)


def as_update(ops):
    """(handles u32, records, live u8) of one step, as r3_update_point_light_sources takes them."""
    handles = np.array([h for h, _ in ops], dtype=np.uint32)
    live = np.array([0 if l is None else 1 for _, l in ops], dtype=np.uint8)
    return handles, records([l for _, l in ops]), live


def same_buffer(a: bytes, b: bytes) -> bool:
    """Two ShaderPointLightBuffers equal bit for bit, any NaN equal to any NaN (the NaN payloads are not part of the rule)."""
    if len(a) != len(b):
        return False
    x, y = np.frombuffer(a, dtype=np.uint32), np.frombuffer(b, dtype=np.uint32)
    fx, fy = x.view(np.float32), y.view(np.float32)
    return bool(np.all((x == y) | (np.isnan(fx) & np.isnan(fy))))
