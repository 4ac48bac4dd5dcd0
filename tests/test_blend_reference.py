"""The blend (transparent) routine against the exact reference of tests/blend_reference.py.

Scenes are drawn through the orthographic camera of tests/raster_scenes.py (world x, y = framebuffer pixels, world z = depth), so
the snapped vertices and the vertex depths the kernels see are known exactly.  Every transparent layer is an object of its own with
an unlit material of its own colour and alpha: layer r of n is translated by 16 (n - r) pixels along x (the mesh is offset by the
opposite, so the snapped vertices do not move), which makes the back-to-front sort draw it r-th.  A swapped pair of layers changes
the bits, so the equality with the reference also checks the draw order.

The CPU part pins the reference to the oracle backend, bit for bit.  The GPU part compares the rgba16f target, the f32 parity
target, the depth and forward_stats()[3] with the reference (identical) and with the oracle, at one and four samples, over two
frames (the second draws the predicted list and culls the residual against the hi-Z), with device and host batching."""
from dataclasses import dataclass, field
from typing import List, Tuple

import numpy as np
import pytest

import blend_case
import blend_reference as bref
import raster_reference as ref
import raster_scenes as rscenes
from rend3_b200 import glam
from rend3_b200.backend import CAMERA_VIEWPORT
from rend3_b200.routines import BaseRenderGraphSettings
from rend3_b200.runner import TestRunner
from rend3_b200.world import BLEND, LEFT, DirectionalLight, MeshBuilder, Object, PbrMaterial

from oracle import load_oracle_backend

f32 = np.float32
CLEAR = rscenes.CLEAR
LAYER_STEP = 16.0            # pixels of x translation between the objects of consecutive layers
POOL_MIN = 1 << 20           # r3_raster.cu:764: the fragment pool starts at max(2^20, W * H * S) nodes
COLLECT_LAUNCHES = 3         # r3_raster.cu:669, 715, 719: region prefix, set-up and band kernel of one collect pass


# ------------------------------------------------------------------ scenes
@dataclass
class Part:
    """Triangles in pixels (n, 3, 2), positively oriented in the y-down framebuffer, with f32 vertex depths (n, 3)."""
    tris: np.ndarray
    z: np.ndarray
    colour: Tuple[float, float, float, float]
    lit: bool = False

    def draw(self):
        return bref.Draw(ref.snap_exact(self.tris), np.asarray(self.z, dtype=f32), self.colour)


@dataclass
class Scene:
    width: int
    height: int
    opaque: List[Part]
    layers: List[Part]                   # transparent objects in draw order (back to front)
    shift: List[float] = field(default_factory=list)   # per-layer y translation in pixels (moved frames)

    def expected(self, samples, rows=None):
        layers = [bref.Draw(l.draw().tris + np.array([0, int(s * ref.SUBPIXEL)]), l.draw().z, l.colour)
                  for l, s in zip(self.layers, self.shift or [0.0] * len(self.layers))]
        return bref.expected(self.width, self.height, samples, CLEAR, [o.draw() for o in self.opaque], layers, rows)


def part(tris, z, colour, lit=False):
    t = np.asarray(tris, dtype=np.float64).reshape(-1, 3, 2)
    z = np.asarray(z, dtype=f32)
    z = np.repeat(z[:, None], 3, axis=1) if z.ndim == 1 else z.reshape(-1, 3)
    assert np.all(ref.signed_area(ref.snap_exact(t)) > 0), "triangles must face the camera"
    return Part(t, z, tuple(float(f32(c)) for c in colour), lit)


def full_cover(width, height):
    """One triangle that covers every sample of the target (its vertices stay well inside the guard band)."""
    return [((-width, -height), (3.0 * width, -height), (-width, 3.0 * height))]


def colours(n, seed):
    rng = np.random.default_rng(seed)
    c = rng.uniform(0.0, 1.0, (n, 4))
    c[:, 3] = rng.uniform(0.05, 0.95, n)
    return c.astype(f32)


def deep_scene(n, order, width=64, height=64):
    """n full-cover layers over an opaque full-cover background at depth 0.1."""
    z = np.sort(rscenes.distinct_depths(n, seed=n))
    if order == "front_to_back":
        z = z[::-1]
    elif order == "interleaved":
        z = np.random.default_rng(100 + n).permutation(z)
    cols = colours(n, seed=n)
    cover = full_cover(width, height)
    return Scene(width, height, [part(cover, [0.1], (0.8, 0.6, 0.2, 1.0))], [part(cover, [z[i]], cols[i]) for i in range(n)])


def partial_scene(seed=1, n_layers=6):
    """Opaque jittered-grid tiles (four objects of their own colours) under layers of boundary-scene triangles (edges and vertices on
    sample points, overlapping inside one object at interleaved depths) and one layer of a jittered grid: the samples of a 4x pixel
    hold different layer sets and different opaque owners, and some layers lie behind some tiles."""
    size = 256
    grid = rscenes.jittered_grid(size, 16, seed=seed)
    tris, _ = rscenes.boundary_scene(size, seed=seed)
    cover = rscenes.jittered_grid(size, 64, seed=seed + 7)
    z = rscenes.distinct_depths(len(grid) + len(tris) + len(cover), seed=seed)
    zg, zt, zc = z[:len(grid)], z[len(grid):len(grid) + len(tris)], z[len(grid) + len(tris):]
    oc = colours(4, seed=seed + 50)
    oc[:, 3] = 1.0
    opaque = [part(grid[k::4], zg[k::4], oc[k]) for k in range(4)]
    lc = colours(n_layers + 1, seed=seed + 60)
    layers = [part(tris[k::n_layers], zt[k::n_layers], lc[k]) for k in range(n_layers)]
    layers.insert(n_layers // 2, part(cover, zc, lc[n_layers]))
    return Scene(size, size, opaque, layers)


A_TRI = [((8.5, 8.5), (56.5, 8.5), (8.5, 56.5))]
B_TRI = [((20.25, 4.5), (60.5, 40.75), (20.25, 60.5))]
C_TRI = [((40.5, 56.5), (62.0, 56.5), (62.0, 63.75))]


def tie_scene():
    """Equal depths from bit-identical geometry: a transparent copy of the opaque triangle A at A's depth (the collect's >=), the
    triangle B twice in one mesh and once more in the next object (the apply's GreaterEqual between layers), and a layer at depth 0
    where no opaque triangle lies (over the clear depth)."""
    cols = colours(4, seed=9)
    opaque = [part(A_TRI, [0.5], (0.2, 0.7, 0.4, 1.0))]
    layers = [part(A_TRI, [0.5], cols[0]), part(B_TRI * 2, [0.625, 0.625], cols[1]), part(B_TRI, [0.625], cols[2]), part(C_TRI, [0.0], cols[3])]
    return Scene(64, 64, opaque, layers)


def behind_scene():
    """An opaque full-cover plane at 0.5; a layer wholly behind it, and sloped layers whose plane crosses it."""
    cover = full_cover(64, 64)
    cols = colours(3, seed=11)
    sloped = [((-4.0, -4.0), (70.0, 2.0), (10.0, 68.0))]
    other = [((60.0, -2.0), (66.0, 66.0), (-3.0, 30.0))]
    layers = [part(cover, [0.3], cols[0]), part(sloped, [[0.2, 0.9, 0.55]], cols[1]), part(other, [[0.8, 0.35, 0.45]], cols[2])]
    return Scene(64, 64, [part(cover, [0.5], (0.3, 0.3, 0.9, 1.0))], layers)


DEPTHS = [1, 2, 7, 8, 9, 31, 32, 33, 64]
ORDERS = ["back_to_front", "front_to_back", "interleaved"]
SCENES = {
    **{f"deep_{n}_{o}": (lambda n=n, o=o: deep_scene(n, o)) for n in DEPTHS for o in ORDERS},
    "partial": partial_scene,
    "ties": tie_scene,
    "behind": behind_scene,
    "narrow_16x64": lambda: deep_scene(9, "interleaved", 16, 64),
    "narrow_8x256": lambda: deep_scene(9, "interleaved", 8, 256),
}


def mesh(tris, z, offset=(0.0, 0.0), uv=False):
    t = np.asarray(tris, dtype=np.float64).reshape(-1, 3, 2) - np.asarray(offset)
    pos = np.zeros((3 * len(t), 3), dtype=f32)
    pos[:, :2] = t.reshape(-1, 2)
    pos[:, 2] = np.asarray(z, dtype=f32).reshape(-1)
    assert np.array_equal(pos[:, :2].astype(np.float64), t.reshape(-1, 2)), "positions must be exact in f32"
    normals = np.tile(np.array([0.0, 0.0, -1.0], dtype=f32), (len(pos), 1))
    b = MeshBuilder.new(pos, LEFT).with_vertex_normals(normals)
    if uv:
        b = b.with_vertex_texture_coordinates_0((pos[:, :2] + np.asarray(offset, dtype=f32)) / f32(16.0))
    return b.build()


def build(backend, scene: Scene, texture=None, light=False):
    r = TestRunner(backend, LEFT)
    tex = r.renderer.add_texture_2d(texture) if texture is not None else None
    for o in scene.opaque:
        mat = PbrMaterial(albedo_value=o.colour, unlit=not o.lit, albedo_texture=tex if o.lit else None)
        r.renderer.add_object(Object(r.renderer.add_mesh(mesh(o.tris, o.z, uv=tex is not None and o.lit)), r.renderer.add_material(mat), glam.identity()))
    r.layers = []
    n = len(scene.layers)
    for rank, l in enumerate(scene.layers):
        tx = LAYER_STEP * (n - rank)
        mat = r.renderer.add_material(PbrMaterial(albedo_value=l.colour, unlit=True, transparency=BLEND))
        m = glam.from_translation((tx, 0.0, 0.0))
        h = r.renderer.add_object(Object(r.renderer.add_mesh(mesh(l.tris, l.z, offset=(tx, 0.0))), mat, m))
        # an added object is located at its bounding sphere's centre (object.rs:256), a moved one at its translation (object.rs:306):
        # setting the same transform again locates it at (tx, 0, 0), whatever its mesh
        r.renderer.set_object_transform(h, m)
        r.layers.append((h, tx))
    last = len(r.renderer.objects) - 1
    if last > 1 and last & (last - 1) == 0:
        # FreelistDerivedBuffer::use_index grows the object buffer on `index > reserved` (buffer.rs:48-54): an object whose handle is
        # a power of two past the last growth is left out of the buffer.  One more object, off-screen, keeps every layer in it.
        off = [((-1000.0, -1000.0), (-990.0, -1000.0), (-1000.0, -990.0))]
        r.renderer.add_object(Object(r.renderer.add_mesh(mesh(off, [0.5, 0.5, 0.5])), r.renderer.add_material(PbrMaterial(unlit=True)), glam.identity()))
    if light:
        r.renderer.add_directional_light(DirectionalLight(color=(1, 1, 1), intensity=2.0, direction=(0.3, -0.4, 1.0), distance=2.0 * scene.width,
                                                          resolution=256))
    r.renderer.set_camera_data(rscenes.ortho_camera(scene.width, scene.height))
    return r


def draw(r, scene, samples, frame, rows=None, srgb_target=True):
    ev = r.renderer.evaluate()
    r.last_eval = ev
    r.base_rendergraph.add_to_graph(ev, (scene.width, scene.height), samples, BaseRenderGraphSettings(clear_color=CLEAR), srgb_target=srgb_target,
                                    upload=frame == 0 or rows is not None, scissor_rows=rows)


def move_layers(r, scene, dy):
    """Translate every layer by dy pixels along y (a whole number of pixels: the snapped vertices stay exact)."""
    for h, tx in r.layers:
        r.renderer.set_object_transform(h, glam.from_translation((tx, float(dy), 0.0)))
    scene.shift = [float(dy)] * len(scene.layers)


# ------------------------------------------------------------------ checks
def read(b):
    return b.readback_hdr_f16().astype(f32), b.readback_hdr_f32(), b.readback_depth(), b.forward_stats()[3]


def assert_frame(b, want: bref.Result, what, mask=None):
    hdr16, hdr32, depth, n = read(b)
    m = np.ones(depth.shape, dtype=bool) if mask is None else mask
    for name, got, exp in (("rgba16f", hdr16, want.hdr16), ("parity f32", hdr32, want.hdr32), ("depth", depth, want.depth)):
        g, e = got[m].view(np.uint32), exp[m].view(np.uint32)
        bad = g != e
        if bad.ndim > 1:
            bad = bad.any(axis=-1)
        assert not bad.any(), f"{what}: {np.count_nonzero(bad)} pixels of the {name} target differ from the reference, first at {np.argwhere(m)[np.argmax(bad)]}: " \
                              f"{got[m][np.argmax(bad)]} against {exp[m][np.argmax(bad)]}"
    if mask is None:
        assert n == want.n_blended, f"{what}: forward_stats()[3] = {n}, the reference blends {want.n_blended}"


def assert_same(a, b, what):
    for name, x, y in zip(("rgba16f", "parity f32", "depth"), read(a)[:3], read(b)[:3]):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), f"{what}: {name} differs"
    assert a.forward_stats()[3] == b.forward_stats()[3], what


# ------------------------------------------------------------------ CPU: the reference against the oracle
@pytest.mark.parametrize("samples", [1, 4])
@pytest.mark.parametrize("name", list(SCENES))
def test_reference_matches_oracle(name, samples):
    """The oracle's frame equals the reference bit for bit: rgba16f, parity target, depth and the blended count."""
    scene = SCENES[name]()
    want = scene.expected(samples)
    assert want.n_blended > 0
    orc = load_oracle_backend()
    r = build(orc, scene)
    for frame in range(2):
        draw(r, scene, samples, frame)
        assert_frame(orc, want, f"oracle {name} {samples}x frame {frame}")
        for srgb in (True, False):
            orc.tonemap(srgb)
            bref.assert_blit(orc.readback_ldr(), want.hdr16, srgb, f"oracle {name} blit srgb={srgb}")


def test_reference_scenes_reach_their_cases():
    """The scenes exercise what they are named for, in the reference itself."""
    for samples in (1, 4):
        d = deep_scene(9, "front_to_back").expected(samples)
        assert d.n_blended == 64 * 64 * samples and d.n_nodes == 9 * 64 * 64 * samples      # only the nearest blends, all are collected
        b = deep_scene(9, "back_to_front").expected(samples)
        assert b.n_blended == b.n_nodes == 9 * 64 * 64 * samples
        t = tie_scene()
        tw = t.expected(samples)
        covered = sum(len(ry) for l in t.layers for ry, _, _, _, _ in bref.fragments([l.draw()], 64, 64, samples))
        assert tw.n_blended == covered, "every tied fragment blends"
        h = behind_scene()
        hw = h.expected(samples)
        only_behind = bref.expected(64, 64, samples, CLEAR, [o.draw() for o in h.opaque], [h.layers[0].draw()])
        assert only_behind.n_nodes == 0 and not only_behind.blended.any()
        full = 64 * 64 * samples
        assert 0.2 * full < hw.n_blended < 1.6 * full, "the sloped layers are cut along the opaque plane"
        p = partial_scene().expected(samples)
        assert p.n_nodes > p.n_blended > 1000
        if samples == 4:
            s = p.samples_f16
            assert np.count_nonzero((s != s[:, :, :1]).any(axis=(2, 3)) & p.blended) > 200, "no 4x pixel with different samples"


def test_alpha_invariants_on_the_oracle():
    """Alpha 0 leaves the rgba16f target unchanged and alpha 1 replaces every covered sample, over lit and textured opaque content."""
    for samples in (1, 4):
        check_alpha_invariants(load_oracle_backend, samples, "oracle")


# ------------------------------------------------------------------ alpha 0 / alpha 1 over content the reference does not restate
def opaque_content(kind):
    """Lit or textured opaque tiles, or nothing but the skybox."""
    tiles = rscenes.jittered_grid(64, 16, seed=3)
    z = rscenes.distinct_depths(len(tiles), seed=3) * f32(0.5)
    if kind == "sky":
        return [], None
    return [part(tiles[k::2], z[k::2], (0.9, 0.5, 0.3, 1.0), lit=True) for k in range(2)], (rscenes.cutout_texture() if kind == "textured" else None)


def alpha_scene(kind, alpha):
    opaque, tex = opaque_content(kind)
    tris = rscenes.jittered_grid(64, 8, seed=5)[::3]
    layer = part(full_cover(64, 64) if alpha == 1.0 else tris, [0.9] * (1 if alpha == 1.0 else len(tris)), (0.25, 0.5, 0.75, alpha))
    return Scene(64, 64, opaque, [layer]), Scene(64, 64, opaque, []), tex


def sky_faces():
    rng = np.random.default_rng(2)
    return [rng.integers(0, 256, (8, 8, 4), dtype=np.uint8) for _ in range(6)]


def render_alpha(make_backend, scene, tex, kind, samples):
    b = make_backend()
    r = build(b, scene, texture=tex, light=kind != "sky")
    if kind == "sky":
        r.renderer.set_skybox(sky_faces(), srgb=False)
    frames = []
    for frame in range(2):
        draw(r, scene, samples, frame)
        frames.append(read(b))
    return b, frames


def check_alpha_invariants(make_backend, samples, what, kinds=("lit", "textured", "sky")):
    for kind in kinds:
        for alpha in (0.0, 1.0):
            with_layer, without, tex = alpha_scene(kind, alpha)
            _, got = render_alpha(make_backend, with_layer, tex, kind, samples)
            _, base = render_alpha(make_backend, without, tex, kind, samples)
            layer = with_layer.layers[0].draw()
            zl = np.zeros((64, 64, samples), dtype=np.uint32)
            for ry, rx, k, z, _ in bref.fragments([layer], 64, 64, samples):
                zl[ry, rx, k] = z
            for frame in range(2):
                h16, h32, depth, n = got[frame]
                b16, b32, bdepth, _ = base[frame]
                tag = f"{what} {kind} alpha {alpha} {samples}x frame {frame}"
                zb = bdepth.view(np.uint32)
                if alpha == 0.0:
                    assert np.array_equal(h16.view(np.uint32), b16.view(np.uint32)), f"{tag}: an invisible layer changed the rgba16f target"
                    covered = (zl != 0).any(axis=2)
                    if samples == 4:
                        assert np.array_equal(h32.view(np.uint32), b32.view(np.uint32)), f"{tag}: parity target"
                        assert covered.sum() > 100
                    else:
                        assert np.array_equal(h32[covered], bref.f16(b32[covered])), f"{tag}: a blended 1x pixel holds the f16 value"
                        assert np.array_equal(h32[~covered], b32[~covered])
                        dz = np.where(zl[..., 0] >= zb, zl[..., 0], zb)
                        assert np.array_equal(depth.view(np.uint32), dz), f"{tag}: depth"
                    assert n > 0
                else:
                    want = np.append(bref.f16(np.asarray(with_layer.layers[0].colour[:3], dtype=f32)), f32(1.0))
                    assert np.array_equal(h16.reshape(-1, 4), np.broadcast_to(want, (64 * 64, 4))), f"{tag}: an opaque layer must replace every sample"
                    assert np.array_equal(h32.reshape(-1, 4), np.broadcast_to(want, (64 * 64, 4))), f"{tag}: parity target"
                    assert np.array_equal(depth.view(np.uint32), zl.min(axis=2)), f"{tag}: depth"
                    assert n == 64 * 64 * samples


# ------------------------------------------------------------------ GPU
@pytest.fixture()
def cuda():
    from rend3_b200.backend import load_cuda_backend

    b = load_cuda_backend(0, parity_target=True)
    yield b
    b.close()


def cuda_backend():
    from rend3_b200.backend import load_cuda_backend

    return load_cuda_backend(0, parity_target=True)


def set_batching(monkeypatch, host):
    if host:
        monkeypatch.setenv("R3_HOST_BATCHING", "1")
    else:
        monkeypatch.delenv("R3_HOST_BATCHING", raising=False)


@pytest.mark.gpu
@pytest.mark.parametrize("host", [False, True], ids=["device_batching", "host_batching"])
@pytest.mark.parametrize("samples", [1, 4])
@pytest.mark.parametrize("name", list(SCENES))
def test_blend_matches_reference(cuda, monkeypatch, name, samples, host):
    """Two frames of each scene: identical to the reference and to the oracle, and the blit of the result equal to blit.wgsl."""
    set_batching(monkeypatch, host)
    scene = SCENES[name]()
    want = scene.expected(samples)
    orc = load_oracle_backend()
    runners = [build(b, scene) for b in (cuda, orc)]
    for frame in range(2):
        for r in runners:
            draw(r, scene, samples, frame)
        assert (cuda.batching_info(CAMERA_VIEWPORT)["path"] == "host") == host
        assert_frame(cuda, want, f"{name} {samples}x frame {frame}")
        assert_same(cuda, orc, f"{name} {samples}x frame {frame} against the oracle")
        for srgb in (True, False):
            cuda.tonemap(srgb)
            bref.assert_blit(cuda.readback_ldr(), want.hdr16, srgb, f"{name} blit srgb={srgb}")


@pytest.mark.gpu
@pytest.mark.parametrize("samples", [1, 4])
def test_alpha_invariants(samples):
    """Alpha 0 / alpha 1 over lit and textured opaque tiles and over the skybox: the 4x re-shade of the opaque samples under a
    transparent layer must reproduce the resolve's samples bit for bit, on both frames."""
    check_alpha_invariants(cuda_backend, samples, "cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("samples", [1, 4])
def test_clipped_transparent_quad(cuda, samples):
    """A blended quad reaching 400x past the guard band: every sample is blended exactly once although its clipped sub-triangles
    share one record."""
    r = rscenes.build(cuda, 256, 256, rscenes.GUARD_QUAD, [0.5, 0.5], transparency=BLEND)
    orc = load_oracle_backend()
    ro = rscenes.build(orc, 256, 256, rscenes.GUARD_QUAD, [0.5, 0.5], transparency=BLEND)
    for frame in range(2):
        rscenes.draw(r, 256, 256, samples)
        rscenes.draw(ro, 256, 256, samples)
        assert cuda.forward_stats()[3] == 256 * 256 * samples
        want = np.array(blend_case.blend(rscenes.COLOUR, [blend_case.f16(v) for v in CLEAR]), dtype=f32)
        hdr = cuda.readback_hdr_f32().reshape(-1, 4)
        assert np.array_equal(hdr, np.broadcast_to(want, hdr.shape)), f"{np.count_nonzero((hdr != want).any(axis=1))} pixels are not one layer"
        assert_same(cuda, orc, f"guard quad frame {frame}")


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [(13, 37), (24, 61)])
@pytest.mark.parametrize("samples", [1, 4])
def test_blend_scissor_rows(cuda, samples, rows):
    """A full frame, then a frame with every layer moved down 8 rows drawn in a band of rows: inside equals the reference and a fresh
    full frame of the moved scene, outside keeps the first frame."""
    scene = partial_scene(seed=2)
    r = build(cuda, scene)
    draw(r, scene, samples, 0)
    first = read(cuda)
    move_layers(r, scene, 8)
    draw(r, scene, samples, 1, rows=rows)
    inside = np.zeros((scene.height, scene.width), dtype=bool)
    inside[rows[0]:rows[1]] = True
    want = scene.expected(samples, rows)
    assert_frame(cuda, want, f"band {rows} {samples}x", mask=inside)
    assert cuda.forward_stats()[3] == want.n_blended
    got = read(cuda)
    for g, f, name in zip(got[:3], first[:3], ("rgba16f", "parity f32", "depth")):
        assert np.array_equal(g[~inside].view(np.uint32), f[~inside].view(np.uint32)), f"{name}: rows outside the band were written"
    fresh = cuda_backend()
    rf = build(fresh, scene)
    move_layers(rf, scene, 8)
    draw(rf, scene, samples, 0)
    for g, f, name in zip(got[:3], read(fresh)[:3], ("rgba16f", "parity f32", "depth")):
        assert np.array_equal(g[inside].view(np.uint32), f[inside].view(np.uint32)), f"{name}: rows inside differ from a full frame"
    fresh.close()


# ------------------------------------------------------------------ the fragment-pool retry
def one_sample_triangle(covering):
    """A triangle around the centre of pixel (10, 10) that covers exactly that sample at one sample and sample 1 at four (and passes the
    small-primitive cull), or, with covering=False, a triangle that covers no sample."""
    return [((10.25, 10.25), (11.25, 10.25), (10.25, 11.25))] if covering else [((10.25, 10.25), (10.4375, 10.25), (10.25, 10.4375))]


def pool_scene(width, height, n_full, covering):
    cover = full_cover(width, height)
    z = np.sort(rscenes.distinct_depths(n_full + 1, seed=n_full))
    cols = colours(n_full + 1, seed=3)
    layers = [part(cover, [z[i]], cols[i]) for i in range(n_full)]
    layers.append(part(one_sample_triangle(covering), [z[n_full]], cols[n_full]))
    return Scene(width, height, [], layers)


def launches_per_frame(b, r, scene, samples, frames=2, rows=None):
    out = []
    for frame in range(frames):
        before = b.launch_count()
        draw(r, scene, samples, frame, rows=rows if frame else None)
        b.sync()
        out.append(b.launch_count() - before)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("frame_graph", [False, True])
@pytest.mark.parametrize("width,height,samples,n_full", [(256, 256, 1, 16), (1024, 512, 4, 1)])
def test_fragment_pool_retry(monkeypatch, width, height, samples, n_full, frame_graph):
    """Exactly the initial pool's node count does not retry; one node more retries the collect once (one more collect pass of
    launches) and gives the reference's image; the next frame fits the grown pool.  A recorded frame is flushed by the readback."""
    monkeypatch.setenv("R3_FRAME_GRAPH", "1" if frame_graph else "0")
    pool = max(POOL_MIN, width * height * samples)
    counts = {}
    for covering in (False, True):
        scene = pool_scene(width, height, n_full, covering)
        want = scene.expected(samples)
        assert want.n_nodes == pool + (1 if covering else 0), (want.n_nodes, pool)
        b = cuda_backend()
        r = build(b, scene)
        counts[covering] = launches_per_frame(b, r, scene, samples)
        assert_frame(b, want, f"pool covering={covering}")
        if frame_graph:
            # the collect's readback drains the stream in the middle of each recorded frame: both frames are flushed there (or earlier)
            st = b.frame_graph_stats()
            assert st["frames"] == 2 and st["flushed"] == 2, f"frame graph stats {st}"
        b.close()
    assert counts[True][0] == counts[False][0] + COLLECT_LAUNCHES, f"one retried collect pass: {counts}"
    assert counts[True][1] == counts[False][1], f"the grown pool holds the second frame: {counts}"


@pytest.mark.gpu
@pytest.mark.parametrize("samples", [1])
def test_fragment_pool_counts_only_the_band(samples):
    """17 full-cover layers at 256x256 overflow the initial pool over the whole target, but not in a band of 24 rows: the band's
    frame must not retry."""
    scene = pool_scene(256, 256, 17, False)
    assert scene.expected(samples).n_nodes > POOL_MIN and scene.expected(samples, (13, 37)).n_nodes < POOL_MIN
    counts = []
    for rows in (None, (13, 37)):
        b = cuda_backend()
        r = build(b, scene)
        before = b.launch_count()
        draw(r, scene, samples, 0, rows=rows)
        b.sync()
        counts.append(b.launch_count() - before)
        if rows is not None:
            inside = np.zeros((256, 256), dtype=bool)
            inside[rows[0]:rows[1]] = True
            assert_frame(b, scene.expected(samples, rows), "band pool", mask=inside)
        b.close()
    assert counts[0] == counts[1] + COLLECT_LAUNCHES, f"the whole target retries, the band does not: {counts}"
