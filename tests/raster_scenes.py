"""Scenes for the rasteriser tests whose snapped vertices are known exactly.

One object with an identity transform seen through a raw orthographic camera glam.orthographic_lh(0, W, H, 0, 0, 1): world x, y
are framebuffer pixels (y down) and world z is the depth.  With W and H powers of two and every position a multiple of 1/256 pixel,
the f32 bake, the divide and the snap are exact, so tests/raster_reference.py knows the integers the kernels see.  Every triangle
has its own three vertices and its own constant z > 0 (reverse-Z clears to 0), so the depth buffer names the front triangle at each
pixel, and triangles are oriented to face the camera (positive area in the y-down framebuffer)."""
import numpy as np

import raster_reference as ref
from rend3_b200 import glam
from rend3_b200.routines import BaseRenderGraphSettings
from rend3_b200.runner import TestRunner
from rend3_b200.world import CUTOUT, LEFT, OPAQUE, Camera, DirectionalLight, MeshBuilder, Object, PbrMaterial, Texture

CLEAR = (0.1, 0.2, 0.3, 1.0)
COLOUR = (0.7, 0.2, 0.9, 0.25)   # unlit; its alpha only matters for the blend routine
# a quad twice across the target in both directions would not be clipped; this one reaches 400x past the guard band
GUARD_QUAD = [((-1.0e5, -1.0e5), (1.0e5, -1.0e5), (1.0e5, 1.0e5)), ((-1.0e5, -1.0e5), (1.0e5, 1.0e5), (-1.0e5, 1.0e5))]


def ortho_camera(width, height):
    return Camera(("raw", glam.orthographic_lh(0.0, float(width), float(height), 0.0, 0.0, 1.0)), glam.identity())


def oriented(tris_px):
    """Triangles in pixels with the last two vertices swapped where needed, so every one faces the camera."""
    t = np.asarray(tris_px, dtype=np.float64).reshape(-1, 3, 2).copy()
    a = (t[:, 1, 0] - t[:, 0, 0]) * (t[:, 2, 1] - t[:, 0, 1]) - (t[:, 2, 0] - t[:, 0, 0]) * (t[:, 1, 1] - t[:, 0, 1])
    t[a < 0, 1], t[a < 0, 2] = t[a < 0, 2].copy(), t[a < 0, 1].copy()
    return t


def distinct_depths(n, seed=0):
    """n distinct f32 depths in [0.25, 0.75], far enough apart (>= 2^-12 / n) that a depth read back names its triangle."""
    z = (0.25 + 0.5 * (np.arange(n) + 1) / (n + 1)).astype(np.float32)
    return np.random.default_rng(seed).permutation(z)


def mesh(tris_px, z, uv=False):
    t = np.asarray(tris_px, dtype=np.float64).reshape(-1, 3, 2)
    pos = np.zeros((3 * len(t), 3), dtype=np.float32)
    pos[:, :2] = t.reshape(-1, 2)
    pos[:, 2] = np.repeat(np.asarray(z, dtype=np.float32), 3)
    assert np.array_equal(pos[:, :2].astype(np.float64), t.reshape(-1, 2)), "positions must be exact in f32"
    normals = np.tile(np.array([0.0, 0.0, -1.0], dtype=np.float32), (len(pos), 1))
    b = MeshBuilder.new(pos, LEFT).with_vertex_normals(normals)
    if uv:
        b = b.with_vertex_texture_coordinates_0(pos[:, :2] / np.float32(16.0))   # the cutout texture repeats every 16 pixels
    return b.build()


def cutout_texture():
    """16x16 texels whose alpha alternates above and below the 0.5 cutout threshold in 4-texel blocks."""
    data = np.full((16, 16, 4), 255, dtype=np.uint8)
    y, x = np.mgrid[0:16, 0:16]
    data[..., 3] = np.where(((x // 4) + (y // 4)) % 2 == 0, 230, 40)
    return Texture(data, srgb=False, mips="none")


def build(backend, width, height, tris_px, z, transparency=OPAQUE, cutout=False, shadow=False):
    """A TestRunner drawing `tris_px` (pixels, (n, 3, 2)) at depths `z` as one object."""
    r = TestRunner(backend, LEFT)
    if cutout:
        tex = r.renderer.add_texture_2d(cutout_texture())
        mat = r.renderer.add_material(PbrMaterial(albedo_texture=tex, albedo_value=(1.0, 1.0, 1.0, 1.0), transparency=CUTOUT, alpha_cutout=0.5,
                                                  sample_type="nearest"))
    else:
        mat = r.renderer.add_material(PbrMaterial(albedo_value=COLOUR, unlit=True, transparency=transparency))
    r.object = r.renderer.add_object(Object(r.renderer.add_mesh(mesh(oriented(tris_px), z, uv=cutout)), mat, glam.identity()))
    if shadow:
        # the light shines along +z, onto the triangles' back faces, which the shadow passes draw; its camera is centred on the
        # viewer's origin, so a distance of 2 x width covers the scene, at one texel per pixel with a 2 x width resolution
        r.renderer.add_directional_light(DirectionalLight(color=(1, 1, 1), intensity=1.0, direction=(0.0, 0.0, 1.0), distance=2.0 * width,
                                                          resolution=2 * width))
    r.renderer.set_camera_data(ortho_camera(width, height))
    return r


def draw(r, width, height, samples):
    r.render_frame(resolution=(width, height), samples=samples, settings=BaseRenderGraphSettings(clear_color=CLEAR))


def snapped(tris_px):
    """The 24.8 integers the kernels see, with the exactness of the f32 path asserted (in float64)."""
    return ref.snap_exact(oriented(tris_px))


# ------------------------------------------------------------------ scenes
def _box_triangles(w, h, x, y):
    """The four right triangles with vertices on the pixel centres of a w x h pixel box at pixel (x, y): their pixel box is
    exactly w x h with one sample or four."""
    x0, y0, x1, y1 = x + 0.5, y + 0.5, x + w - 0.5, y + h - 0.5
    c = [(x0, y0), (x1, y0), (x1, y1), (x0, y1)]
    return [(c[k], c[(k + 1) % 4], c[(k + 3) % 4]) for k in range(4)]


BOUNDARY_BOXES = [(8, 8), (16, 4), (4, 16), (32, 2), (13, 5), (5, 13), (33, 2), (32, 32), (32, 33), (33, 32), (60, 40)]


def boundary_scene(size=256, seed=1):
    """Triangles on both sides of every path threshold: pixel boxes of exactly 64 and 65 pixels (8x8, 16x4, 32x2 / 13x5, 33x2),
    32x32 against 32x33 and 33x32, a band-sized box; edge reach of exactly FITS32_REACH and one past it on the inline and the
    cooperative path (a vertex beyond the left or top edge of the target, the only way a vertex can reach farther than the box);
    and triangles with vertices on random sample positions.  Returns (triangles in pixels, labels)."""
    rng = np.random.default_rng(seed)
    tris, labels = [], []
    for w, h in BOUNDARY_BOXES:
        # even pixel offsets: a 2-pixel box spans from y + 0.5 to y + 1.5, which the triangle cull rounds (half to even) apart
        x, y = 2 * int(rng.integers(1, (size - w) // 2 - 1)), 2 * int(rng.integers(1, (size - h) // 2 - 1))
        for k, t in enumerate(_box_triangles(w, h, x, y)):
            tris.append(t)
            labels.append(f"box {w}x{h} corner {k}")
    for reach in (ref.FITS32_REACH, ref.FITS32_REACH + 1):
        for far, n in (("inline", 4), ("coop", 21)):
            # the far vertex sits `reach` sub-pixels from the centre of pixel 0 on one axis, beyond the target's edge
            y = int(rng.integers(2, size - n - 2))
            far_x = (128 - reach) / 256.0
            tris.append(((far_x, y + 0.5), (n - 0.5, y + 0.5), (n - 0.5, y + n - 0.5)))
            labels.append(f"{far} reach {reach} along x")
            x = int(rng.integers(2, size - n - 2))
            tris.append(((x + 0.5, far_x), (x + n - 0.5, n - 0.5), (x + 0.5, n - 0.5)))
            labels.append(f"{far} reach {reach} along y")
    offsets = np.array([(0, 0)] + list(zip(ref.SAMPLE_DX, ref.SAMPLE_DY))) + 128
    for i in range(48):
        span = int(rng.choice([6, 12, 30, 70]))
        ox, oy = rng.integers(0, size - span - 1, 2)
        pts = []
        for _ in range(3):
            px, py = rng.integers(0, span + 1, 2)
            dx, dy = offsets[rng.integers(0, 5)]
            pts.append(((ox + px) + dx / 256.0, (oy + py) + dy / 256.0))
        tris.append(tuple(pts))
        labels.append(f"sample-position triangle {i}")
    t = oriented(tris)
    s = ref.snap_exact(t)
    keep = (ref.signed_area(s) != 0) & ~ref.small_primitive_culled(s)   # the single-sample triangle cull would drop the others
    return t[keep], [l for l, k in zip(labels, keep) if k]


def jittered_grid(size, cell, seed, ties=True):
    """A grid of size/cell squares with jittered interior nodes, each square split in two triangles: the triangles tile the
    target exactly.  With `ties` half of the nodes sit on pixel centres, so edges pass through sample points."""
    rng = np.random.default_rng(seed)
    n = size // cell
    gx, gy = np.meshgrid(np.arange(n + 1) * float(cell), np.arange(n + 1) * float(cell))
    j = cell // 4
    jit = rng.integers(-j * 256, j * 256 + 1, (2, n + 1, n + 1)) / 256.0
    if ties:
        centre = rng.random((n + 1, n + 1)) < 0.5
        jit[:, centre] = np.floor(jit[:, centre]) + 0.5
    interior = np.zeros((n + 1, n + 1), dtype=bool)
    interior[1:-1, 1:-1] = True
    gx = np.where(interior, gx + jit[0], gx)
    gy = np.where(interior, gy + jit[1], gy)
    tris = []
    for i in range(n):
        for k in range(n):
            a, b, c, d = (gx[i, k], gy[i, k]), (gx[i, k + 1], gy[i, k + 1]), (gx[i + 1, k + 1], gy[i + 1, k + 1]), (gx[i + 1, k], gy[i + 1, k])
            tris += [(a, b, c), (a, c, d)] if (i + k) % 2 == 0 else [(a, b, d), (b, c, d)]
    return oriented(tris)


def block_corner_triangles(size=256, n=40, seed=5):
    """Large triangles whose edges pass within a pixel of the corners of the band kernel's 32 x 16 blocks."""
    rng = np.random.default_rng(seed)
    tris = []
    while len(tris) < n:
        cx, cy = rng.integers(1, size // 32) * 32, rng.integers(1, size // 16) * 16
        d = rng.integers(30 * 256, 90 * 256, 2) * rng.choice([-1, 1], 2)
        e = rng.integers(-256, 257, 2)
        a = (cx * 256 + d[0], cy * 256 + d[1])
        b = (cx * 256 - d[0] + e[0], cy * 256 - d[1] + e[1])
        c = (rng.integers(0, size * 256), rng.integers(0, size * 256))
        t = np.clip(np.array([a, b, c]), 0, size * 256 - 1) / 256.0
        s = ref.snap_exact(t)[None]
        if abs(int(ref.signed_area(s)[0])) > 2 * 256 * 256 * 40:
            tris.append(t)
    return oriented(tris)


# ------------------------------------------------------------------ checks against the exact reference
def owners_from_depth(depth, z, max_ulps=8):
    """Index of the triangle whose depth each texel holds (-1 for the clear value 0), asserting it is within `max_ulps` f32 units
    in the last place of that triangle's plane depth: R5 rounds the three weighted terms, nothing more."""
    z = np.asarray(z, dtype=np.float32)
    order = np.argsort(z, kind="stable")
    zs = z[order].astype(np.float64)
    d = depth.ravel().astype(np.float64)
    hi = np.clip(np.searchsorted(zs, d), 0, len(zs) - 1)
    lo = np.clip(hi - 1, 0, len(zs) - 1)
    own = order[np.where(np.abs(d - zs[lo]) <= np.abs(zs[hi] - d), lo, hi)]
    drawn = d != 0.0
    ulps = ref.f32_ulps(depth.ravel()[drawn], z[own[drawn]])
    assert ulps.size == 0 or ulps.max() <= max_ulps, f"a depth is {ulps.max()} ulps from every triangle's plane"
    own = np.where(drawn, own, -1)
    return own.reshape(depth.shape)


def expected_pixel_owners(owner, z):
    """The triangle whose depth the resolved depth buffer holds: with four samples the resolve keeps the minimum over the samples,
    and an uncovered sample (clear depth 0) wins."""
    if owner.shape[2] == 1:
        return owner[..., 0]
    zz = np.where(owner >= 0, np.asarray(z, dtype=np.float64)[np.maximum(owner, 0)], -1.0)
    k = np.argmin(np.where(owner >= 0, zz, -1.0), axis=2)
    return np.take_along_axis(owner, k[..., None], axis=2)[..., 0]


def assert_matches_reference(backend, width, height, tris_px, z, samples, what=""):
    """Covered-sample count (forward_stats()[1]) and the owner of every pixel, read from depth, equal the exact reference's."""
    count, owner = ref.coverage(snapped(tris_px), width, height, samples, z)
    got = backend.forward_stats()[1]
    assert got == count, f"{what}: {got} covered samples, the exact reference counts {count}"
    want = expected_pixel_owners(owner, z)
    have = owners_from_depth(backend.readback_depth(), z)
    bad = have != want
    assert not bad.any(), f"{what}: {np.count_nonzero(bad)} pixels owned by another triangle than in the exact reference, first at {np.argwhere(bad)[0]}"
    return count
