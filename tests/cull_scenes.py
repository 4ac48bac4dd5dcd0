"""Scenes for the triangle-cull tests, fed to `Backend.cull(camera, batches, regions)` through hand-built batch tables.

Exact decision scenes use the tests/raster_scenes.py set-up: a raw orthographic camera glam.orthographic_lh(0, W, H, 0, 0, 1) with an
identity model matrix, a power-of-two target and positions on multiples of 1/256 pixel.  Clip x = px * 2 / W - 1, clip y = 1 - py * 2 / H,
clip z = world z and w = 1 are then exact in f32, and so are the screen boxes, the uv and the depth: f32 and float64 agree exactly.
The hi-Z pyramid those scenes sample comes from occluder rectangles drawn at known constant depths."""
from dataclasses import dataclass, field

import numpy as np

import cull_reference as ref
import raster_scenes
from rend3_b200 import glam
from rend3_b200.backend import CAMERA_VIEWPORT, CB_BAKE
from rend3_b200.layouts import (BATCH_DTYPE, CAMERA_HEADER_DTYPE, NO_PREVIOUS, OBJECT_DTYPE, PCU_MULTISAMPLED, PCU_POSITIVE_AREA_VISIBLE,
                                REGION_DTYPE)

F32 = np.float32
SB_INVOCATIONS = 32768          # one superblock of the compaction: 1024 visibility words
WARP_STRIDE = 132 * 4 * 8       # workgroups between two of one warp's workgroups on a full H100 at 4 CTAs / SM


@dataclass
class Scene:
    objects: np.ndarray                   # OBJECT_DTYPE
    mesh: np.ndarray                      # u32 words
    batches: np.ndarray
    regions: np.ndarray
    labels: list = field(default_factory=list)   # per object


def ortho_header(width, height, flags, n_objects, shadow_index=CAMERA_VIEWPORT, proj=None):
    h = np.zeros((), dtype=CAMERA_HEADER_DTYPE)
    vp = glam.orthographic_lh(0.0, float(width), float(height), 0.0, 0.0, 1.0) if proj is None else proj
    h["view"] = glam.identity().reshape(16)
    h["view_proj"] = np.asarray(vp, dtype=F32).reshape(16)
    h["shadow_index"] = shadow_index
    h["resolution"] = np.array((width, height), dtype=F32)
    h["flags"] = flags
    h["object_count"] = n_objects
    return h


def object_records(n):
    o = np.zeros(n, dtype=OBJECT_DTYPE)
    o["transform"] = glam.identity().reshape(16)
    o["sphere_radius"] = 1.0
    o["enabled"] = 1
    return o


def build_tables(tri_counts, atomic=None, keys=None, prev=None, order=None):
    """Batch and region tables as batching.rs:120-250 lays them out for objects in `order` (default: as given): 256 objects per
    batch, a new region on a key change or a new batch, every object padded to whole workgroups of 256 invocations."""
    n = len(tri_counts)
    order = list(range(n)) if order is None else list(order)
    atomic = [1] * n if atomic is None else atomic
    keys = [0] * n if keys is None else keys
    prev = [NO_PREVIOUS] * n if prev is None else prev
    batches, regions = [], []
    cur = np.zeros((), BATCH_DTYPE)
    cur_obj = cur_inv = base_inv = region_inv = region_obj = 0
    cur_key = keys[order[0]]
    for h in order:
        if keys[h] != cur_key or cur_obj == 256:
            regions.append((len(batches), 0, cur_key))
            cur_key, region_obj, region_inv = keys[h], 0, cur_inv
        if cur_obj == 256:
            cur["total_objects"], cur["total_invocations"], cur["batch_base_invocation"] = cur_obj, cur_inv, base_inv
            batches.append(cur.copy())
            cur = np.zeros((), BATCH_DTYPE)
            base_inv += cur_inv
            cur_inv = cur_obj = region_inv = 0
        r = cur["object_culling_information"][cur_obj]
        r["invocation_start"], r["invocation_end"] = cur_inv, cur_inv + tri_counts[h]
        r["object_id"], r["region_id"] = h, len(regions)
        r["base_region_invocation"], r["local_region_id"] = region_inv, region_obj
        r["previous_global_invocation"], r["atomic_capable"] = prev[h], atomic[h]
        cur_obj += 1
        region_obj += 1
        cur_inv += (tri_counts[h] + 255) // 256 * 256
    regions.append((len(batches), 0, cur_key))
    cur["total_objects"], cur["total_invocations"], cur["batch_base_invocation"] = cur_obj, cur_inv, base_inv
    batches.append(cur.copy())
    reg = np.zeros(len(regions), REGION_DTYPE)
    for i, (j, bg, k) in enumerate(regions):
        reg[i]["job_index"], reg[i]["bind_group_index"], reg[i]["material_key"] = j, bg, k
    return np.array(batches, dtype=BATCH_DTYPE), reg


def regions_atomic(scene):
    """Whether each region's first object is atomic-capable (one material key per region)."""
    out = np.zeros(len(scene.regions), bool)
    for b in scene.batches:
        for info in b["object_culling_information"][:int(b["total_objects"])]:
            if int(info["local_region_id"]) == 0:
                out[int(info["region_id"])] = int(info["atomic_capable"]) == 1
    return out


def total_invocations(batches):
    return int(sum(int(b["total_invocations"]) for b in batches))


# ------------------------------------------------------------------ running a cull and reading it back
def upload(backend, scene):
    backend.set_objects(scene.objects)
    backend.set_mesh_buffer(scene.mesh)


def run_cull(backend, scene, header, camera=CAMERA_VIEWPORT, batches=None, regions=None, settle=True):
    """Bake, cull with the scene's tables, read back what the cull produced.  The residual partition reads back only as long as the
    previous cull's list (InputOutputBuffer: in_elems), although the kernel writes it up to the buffer's capacity.  With `settle`, a
    cull whose predecessor had fewer invocations is run a second time with the same tables so that the whole residual list reads
    back; got["culls"] records it.  Without, the first cull is the one compared, and only the readable part of its residual list."""
    backend.object_uniform_upload(camera, header, CB_BAKE)
    b = scene.batches if batches is None else batches
    r = scene.regions if regions is None else regions
    backend.cull(camera, b, r)
    culls = 1
    if settle and len(backend.readback_indices(camera, 1)) < 3 * total_invocations(b):
        backend.cull(camera, b, r)
        culls = 2
    n = len(scene.objects)
    return dict(words=backend.readback_culling_results(camera, 0).copy(), prev=backend.readback_culling_results(camera, 1).copy(),
                dc_pred=backend.readback_draw_calls(camera, 0).copy(), dc_resid=backend.readback_draw_calls(camera, 1).copy(),
                idx_pred=backend.readback_indices(camera, 0).copy(), idx_resid=backend.readback_indices(camera, 1).copy(),
                mvps=backend.readback_object_matrices(camera, 0, n)["model_view_proj"].reshape(n, 16).copy(), culls=culls, settled=settle)


def read_pyramid(backend, n_levels):
    return [backend.readback_hiz(m).copy() for m in range(n_levels)]


def reference_for(got, scene, header, pyramid):
    """The reference's lists for a cull whose readback is `got`: the same baked MVPs, pyramid and input partition the cull saw."""
    import cull_reference as ref
    return ref.cull_lists(scene.batches, scene.regions, scene.mesh, scene.objects, got["mvps"], header, pyramid, got["prev"])


def assert_matches(got, want, scene, what, ordered=True):
    """Visibility words, both draw-call arrays and their zeroed tail, the defined parts of both index lists (which include the
    non-atomic in-place slots and their INVALID padding)."""
    import cull_reference as ref
    w = want["words"]
    assert np.array_equal(got["words"][:len(w)], w), f"{what}: {np.count_nonzero(got['words'][:len(w)] != w)} visibility words differ"
    for part, key in ((0, "dc_pred"), (1, "dc_resid")):
        d, n = got[key], len(want[key])
        assert d[:n].tobytes() == want[key].tobytes(), f"{what}: draw calls (partition {part}) differ: {d[:n]} against {want[key]}"
        assert not d[n:].view(np.uint8).any(), f"{what}: stray draw calls past the regions (partition {part})"
    if ordered:
        for key, mask in (("idx_pred", "pred_defined"), ("idx_resid", "resid_defined")):
            n = min(len(want[mask]), len(got[key]))          # a residual list read back after a growth is shorter (run_cull)
            m = want[mask][:n]
            h = got[key][:n][m]
            assert np.array_equal(h, want[key][:n][m]), f"{what}: {key}: {np.count_nonzero(h != want[key][:n][m])} defined index words differ"
            if key == "idx_pred" or got.get("settled", True):
                assert n == len(want[mask]) or not want[mask][n:].any(), f"{what}: {key} reads back shorter than its defined part"
    else:
        bad = ref.same_sets(want, got["idx_pred"], got["idx_resid"], regions_atomic(scene))
        assert not bad, f"{what}: regions whose triangle sets differ: {bad[:8]}"


# ------------------------------------------------------------------ one object per triangle, positions in pixels
def triangle_scene(tris_px, z):
    """Every triangle its own object of one triangle, with its own three vertices: (n, 3, 2) pixels, z per triangle (or per vertex)."""
    t = np.asarray(tris_px, dtype=np.float64).reshape(-1, 3, 2)
    n = len(t)
    pos = np.zeros((n, 3, 3), dtype=F32)
    pos[:, :, :2] = t
    pos[:, :, 2] = np.asarray(z, dtype=F32).reshape(n, -1)
    assert np.array_equal(pos[:, :, :2].astype(np.float64), t), "positions must be exact in f32"
    idx = np.arange(3 * n, dtype=np.uint32)
    mesh = np.concatenate([idx, pos.reshape(-1).view(np.uint32)])
    objects = object_records(n)
    objects["first_index"] = np.arange(n) * 3
    objects["index_count"] = 3
    objects["attr_offset"][:, 0] = 4 * 3 * n
    batches, regions = build_tables([1] * n)
    return Scene(objects, mesh, batches, regions)


# ------------------------------------------------------------------ the exact decision scene
EXACT_SIZE = 256
# occluders: x < 128 at depth 0.5 (region A), x >= 128 and y < 128 at 0.25 (region B), x >= 128 and y >= 128 uncovered (region C, 0.0)
OCCLUDERS = [(((0, 0), (128, 0), (128, 256)), 0.5), (((0, 0), (128, 256), (0, 256)), 0.5),
             (((128, 0), (256, 0), (256, 128)), 0.25), (((128, 0), (256, 128), (128, 128)), 0.25)]


def draw_occluders(backend, samples, size=EXACT_SIZE, occluders=OCCLUDERS):
    """Draw the occluders through the rasteriser, rebuild the pyramid from the finished depth buffer and return it."""
    tris = [t for t, _ in occluders]
    r = raster_scenes.build(backend, size, size, tris, [z for _, z in occluders])
    raster_scenes.draw(r, size, size, samples)
    backend.hiz_build()
    return read_pyramid(backend, len(_levels(size, size)))


def _levels(w, h):
    return [(max(w >> i, 1), max(h >> i, 1)) for i in range(int(max(w, h)).bit_length())]


def _box(x0, x1, y0, y1):
    """A right triangle whose screen box is exactly [x0, x1] x [y0, y1]."""
    return ((x0, y0), (x1, y0), (x0, y1))


def exact_decision_triangles():
    """(triangles in pixels, z per triangle, labels).  Every triangle appears in both windings (the mirror follows it)."""
    s = 1.0 / 256
    tris, z, labels = [], [], []

    def add(t, depth, label):
        tris.append(t)
        z.append(depth)
        labels.append(label)
    # det == 0: a repeated vertex, horizontal, vertical and diagonal collinear points
    add(((10, 10), (10, 10), (20, 30)), 0.9, "det0 repeated")
    add(((10, 40), (20, 40), (30, 40)), 0.9, "det0 horizontal")
    add(((50, 10), (50, 20), (50, 35)), 0.9, "det0 vertical")
    add(((130, 130), (131, 131), (133, 133)), 0.9, "det0 diagonal")
    # screen boxes [x + 0.5, x + 1.5] for even and odd x, and one 1/256 step to either side of each end, on both axes
    for x in (40, 41, 170, 171):
        for d0, d1, tag in ((0, 0, "tie"), (-s, 0, "lo-"), (s, 0, "lo+"), (0, -s, "hi-"), (0, s, "hi+")):
            add(_box(x + 0.5 + d0, x + 1.5 + d1, 60, 80), 0.9, f"box x {x} {tag}")
            add(_box(60, 80, x + 0.5 + d0, x + 1.5 + d1), 0.9, f"box y {x} {tag}")
    # longest edge: below 1, exactly 2^k and 2^k + 1/256, larger than the target; centred near the corner of regions A and C so that
    # the mip decides whether the footprint reaches the uncovered region (depth 0.4: behind A's 0.5, in front of C's 0.0)
    add(_box(125.25, 126, 200, 200.75), 0.4, "edge 0.75")
    for k in range(0, 8):
        e = 2.0 ** k
        cx = 128 - 0.75 * e
        for extra, tag in ((0.0, "2^k"), (s, "2^k+")):
            add(_box(cx - e / 2, cx + e / 2 + extra, 190, 190 + min(e, 8)), 0.4, f"edge {tag} k={k}")
    add(_box(-20, 280, 150, 160), 0.4, "edge beyond target")
    # depth at the occluder, one ulp below and one above
    for zz, region in ((0.5, (20, 40)), (0.25, (180, 40))):
        for dz, tag in ((0, "equal"), (-1, "ulp below"), (1, "ulp above")):
            d = np.nextafter(F32(zz), F32(-1 if dz < 0 else 2)) if dz else F32(zz)
            add(_box(region[0], region[0] + 8, region[1], region[1] + 8), float(d), f"depth {tag} {zz}")
    # footprints on and between texels: u * res - 0.5 an integer (one texel) or a quarter past (two texels across the A | C edge)
    add(_box(127, 128, 200, 201), 0.4, "uv integer A")
    add(_box(128, 129, 200, 201), 0.4, "uv integer C")
    add(_box(127.25, 128.25, 200, 201), 0.4, "uv straddles A|C")
    add(_box(127, 128, 127.25, 128.25), 0.4, "uv straddles A|A")
    add(_box(126, 128, 126.5, 128.5), 0.4, "uv integer mip1")
    # partly and wholly off screen
    add(_box(-20, 30, 100, 110), 0.9, "partly off left")
    add(_box(240, 270, -15, 10), 0.45, "partly off top right")
    add(_box(300, 320, 20, 40), 0.9, "wholly off right")
    add(_box(20, 40, -60, -30), 0.9, "wholly off top")
    add(_box(-40, -20, 200, 220), 0.1, "wholly off left")
    t = np.asarray(tris, dtype=np.float64)
    mirrored = t[:, [0, 2, 1]]
    return np.concatenate([t, mirrored]), np.array(z + z, dtype=F32), labels + [l + " mirrored" for l in labels]


EXACT_FLAGS = [0, PCU_POSITIVE_AREA_VISIBLE, PCU_MULTISAMPLED, PCU_POSITIVE_AREA_VISIBLE | PCU_MULTISAMPLED]


# ------------------------------------------------------------------ perspective edges
def perspective_scene(seed=4):
    """Triangles under a reverse-Z perspective camera: one, two or three vertices behind the eye (w < 0), w == 0, NaN, infinite and
    1e30 positions, triangles whose clip w are all exactly 1.0 (the kernel's division skip), and random triangles.  Returns
    (triangles in world space (n, 3, 3), labels, view_proj)."""
    proj = glam.perspective_infinite_reverse_lh(np.float32(np.radians(60.0)), 1.0, 0.5)
    rng = np.random.default_rng(seed)
    tris, labels = [], []
    # w = view z for this projection: z = 1.0 gives w == 1.0 exactly
    for i in range(24):
        xy = rng.uniform(-0.5, 0.5, (3, 2))
        tris.append(np.column_stack([xy, np.ones(3)]))
        labels.append("unit w")
    for n_behind in (1, 2, 3):
        for i in range(8):
            p = np.column_stack([rng.uniform(-3, 3, (3, 2)), rng.uniform(1, 10, 3)])
            p[:n_behind, 2] = -rng.uniform(0.1, 5, n_behind)
            tris.append(p)
            labels.append(f"{n_behind} behind")
    for i in range(8):
        p = np.column_stack([rng.uniform(-3, 3, (3, 2)), rng.uniform(1, 10, 3)])
        p[i % 3, 2] = 0.0
        tris.append(p)
        labels.append("w == 0")
    for bad, tag in ((np.nan, "nan"), (np.inf, "inf"), (-np.inf, "-inf"), (1e30, "1e30"), (-1e30, "-1e30")):
        for comp in range(3):
            p = np.column_stack([rng.uniform(-2, 2, (3, 2)), rng.uniform(2, 6, 3)])
            p[comp % 3, comp] = bad
            tris.append(p)
            labels.append(f"{tag} component {comp}")
    for i in range(200):
        c = np.array([rng.uniform(-8, 8), rng.uniform(-8, 8), rng.uniform(1, 30)])
        tris.append(c + rng.normal(0, rng.choice([0.05, 0.3, 1.5]), (3, 3)))
        labels.append("random")
    return np.asarray(tris, dtype=F32), labels, proj


def world_triangle_scene(tris):
    t = np.asarray(tris, dtype=F32).reshape(-1, 3, 3)
    n = len(t)
    idx = np.arange(3 * n, dtype=np.uint32)
    mesh = np.concatenate([idx, t.reshape(-1).view(np.uint32)])
    objects = object_records(n)
    objects["first_index"] = np.arange(n) * 3
    objects["index_count"] = 3
    objects["attr_offset"][:, 0] = 4 * 3 * n
    batches, regions = build_tables([1] * n)
    return Scene(objects, mesh, batches, regions)


# ------------------------------------------------------------------ structural scenes
def grid_triangles(n, rng, size=EXACT_SIZE):
    """n small triangles at random places on a size x size orthographic target; about a third face away, some miss pixel centres."""
    c = rng.uniform(4, size - 4, (n, 1, 2))
    t = np.round((c + rng.uniform(-3, 3, (n, 3, 2))) * 256) / 256
    return t.astype(F32)


def structural_scene(tri_counts, seed, first_pad=None, pos_pad=None, atomic=None, keys=None, prev=None, tail_words=0):
    """One object per entry of `tri_counts`, each with its own index run and positions, in one mesh buffer:
    [indices of every object, each after `first_pad[i]` filler words] [positions of every object, after `pos_pad[i]` words] [tail].
    Filler words are large non-zero values, so that an index read from the wrong place points far away."""
    rng = np.random.default_rng(seed)
    n = len(tri_counts)
    first_pad = [0] * n if first_pad is None else first_pad
    pos_pad = [0] * n if pos_pad is None else pos_pad
    idx_words, pos_words, objects = [], [], object_records(n)
    cursor = 0
    for i, t in enumerate(tri_counts):
        idx_words.append(np.full(first_pad[i], 0x7FFFFFF0, np.uint32))
        cursor += first_pad[i]
        objects[i]["first_index"] = cursor
        objects[i]["index_count"] = 3 * t
        idx = rng.permutation(3 * t).astype(np.uint32)          # every vertex used once, in a scrambled order
        idx_words.append(idx)
        cursor += 3 * t
    pos_base = cursor
    for i, t in enumerate(tri_counts):
        pos_words.append(np.full(pos_pad[i], 0x7F7FFFFF, np.uint32))
        pos_base += pos_pad[i]
        objects[i]["attr_offset"][0] = 4 * pos_base
        p = np.zeros((3 * t, 3), F32)
        p[:, :2] = grid_triangles(t, rng).reshape(-1, 2)
        p[:, 2] = rng.uniform(0.05, 0.95, 3 * t).astype(F32)
        pos_words.append(p.reshape(-1).view(np.uint32))
        pos_base += 9 * t
    mesh = np.concatenate(idx_words + pos_words + [np.full(tail_words, 0x3F000000, np.uint32)])
    batches, regions = build_tables(list(tri_counts), atomic=atomic, keys=keys, prev=prev)
    return Scene(objects, mesh, batches, regions)


def ragged_scene(seed=11):
    """Objects of 1, 31, 32, 33, 255, 256, 257 and 4097 triangles, first_index and attr_offset[0] at every residue mod 4, a full
    256-object batch whose objects 0, 1, 254 and 255 are non-atomic (blend) with a second material key, and prev offsets that are
    NO_PREVIOUS, in range, and past the input partition (set by the caller for the second frame)."""
    sizes = [1, 31, 32, 33, 255, 256, 257, 4097]
    counts = [sizes[i % len(sizes)] for i in range(256)] + [sizes[i % len(sizes)] for i in range(40)]
    n = len(counts)
    first_pad = [i % 4 for i in range(n)]
    pos_pad = [(i // 4) % 4 for i in range(n)]
    atomic = [0 if i in (0, 1, 254, 255) else 1 for i in range(n)]
    keys = [2 if i in (0, 1, 254, 255) else 0 for i in range(n)]
    return structural_scene(counts, seed, first_pad, pos_pad, atomic, keys)


def big_scene(seed=14, n_objects=3200):
    """About 2.5 M invocations, more than twice the 4224 workgroups a full H100 deals to its warps at once, so every warp tests a second
    and a third workgroup and stages their runs ahead (run_n0): ragged objects, every first_index / attr_offset residue mod 4, and
    every 37th object non-atomic in a region of its own.  Eight one-triangle objects late in the order (far past the first pass of
    the grid, two of them non-atomic) read their indices from the end of the mesh buffer: their first runs end exactly at the
    allocation (mesh_words + 4) or past it, so run_n0 is staged on one side of the guard and rejected on the other.
    Returns (scene, the objects at the end)."""
    sizes = [1, 31, 32, 33, 255, 256, 257, 4097]
    counts = [sizes[i % len(sizes)] for i in range(n_objects)]
    atomic = [0 if i % 37 == 0 else 1 for i in range(n_objects)]
    keys = [2 if a == 0 else 0 for a in atomic]
    s = structural_scene(counts, seed, [i % 4 for i in range(n_objects)], [(i // 4) % 4 for i in range(n_objects)], atomic, keys)
    tail = np.random.default_rng(seed).integers(0, 3, 200).astype(np.uint32)   # vertex ids of one-triangle objects: 0, 1, 2
    end = len(s.mesh) + len(tail)
    s.mesh = np.concatenate([s.mesh, tail])
    ends = [2072, 2368, 2400, 2480, 2560, 2640, 2960, 3192]     # one-triangle objects (i % 8 == 0); 2072, 2368 and 2960 non-atomic
    starts = [end - 96, end - 100, end - 95, end - 94, end - 93, end - 92, end - 40, end - 3]   # the first two staged, the rest rejected
    for o, f in zip(ends, starts):
        assert counts[o] == 1
        s.objects[o]["first_index"] = f
    return s, ends
def superblock_scene(delta, seed=12):
    """Regions that start exactly on a 32768-invocation superblock boundary, end on one and straddle one, with a total of
    4 x 32768 + delta invocations (delta in {-256, 0, 256}).  Every object is its own region."""
    counts = [SB_INVOCATIONS, SB_INVOCATIONS // 2, SB_INVOCATIONS, SB_INVOCATIONS // 2 + SB_INVOCATIONS + delta]
    s = structural_scene(counts, seed, keys=[0, 1, 2, 3])
    assert total_invocations(s.batches) == 4 * SB_INVOCATIONS + delta
    return s


STALE_WORD = 7          # what the larger, earlier mesh buffer holds past the smaller one's end: the valid vertex index 7


def mesh_end_scene(seed=13):
    """Index runs at the end of the mesh allocation.  A fresh context allocates mesh_words + 4 words (r3_set_mesh_buffer, r3_reserve):
    object 0's first staged run (its 16-byte aligned start + 100 words) ends exactly there, object 1's starts four words later and must
    fall back to direct loads.  Object 2's 40 triangles run past mesh_words: triangle 37 is (1, 2, past the end), which robust access
    reads as (1, 2, 0) and passes, while the stale index 7 would make it (1, 2, 7), a back face.  Object 3's first triangle is
    (1, 2, v) with every word of v's position past the end: robust access reads (0, 0, 0) and it passes, while the stale position
    (120, 200) a larger buffer left there makes it a back face.
    Returns (scene, mesh_words, stale) with `stale` the larger buffer to set first, so that the bulk copy reads its words."""
    rng = np.random.default_rng(seed)
    n_pos = 64
    p = np.zeros((n_pos, 3), F32)
    p[:, :2] = grid_triangles(n_pos // 3 + 1, rng).reshape(-1, 2)[:n_pos]
    p[:, 2] = rng.uniform(0.1, 0.9, n_pos)
    p[:3, :2] = ((10, 10), (50, 10), (10, 50))                # vertices 0-2: a triangle that passes, for the runs at the very end
    p[STALE_WORD, :2] = (60, 60)                              # (1, 2, 7): on the other side of the edge from 1 to 2, a back face
    pos = p.reshape(-1).view(np.uint32)
    tri = lambda k: rng.integers(0, n_pos, 3 * k).astype(np.uint32)
    # layout: [positions 192 | object 3's index run | filler | ... | obj0 | obj1 | obj2's indices, running past the end]
    head = np.concatenate([pos, tri(8)])
    end = 4 * ((len(head) + 200) // 4) + 96                    # mesh_words: object 0's aligned start is end - 96
    mesh = np.full(end, 9, np.uint32)                          # filler: the valid vertex index 9
    mesh[:len(head)] = head
    o0, o1, o2 = end - 96, end - 92, end - 3 * 40 + 7         # aligned starts for 0 and 1; object 2's run leaves the buffer
    mesh[o0:o0 + 3], mesh[o1:o1 + 3] = (0, 1, 2), (2, 0, 1)
    mesh[o2:end] = rng.integers(0, n_pos, end - o2)
    mesh[o2 + 111:o2 + 113] = (1, 2)                           # triangle 37: (1, 2, word `end`)
    v = (end + 200 + 2) // 3                                   # object 3's vertex whose position lies wholly past the end
    mesh[len(pos):len(pos) + 3] = (1, 2, v)
    stale = np.full(end + 4096, STALE_WORD, np.uint32)
    stale[:end] = mesh
    stale[3 * v:3 * v + 3] = np.array([120.0, 200.0, 0.5], F32).view(np.uint32)
    objects = object_records(4)
    objects["first_index"] = [o0, o1, o2, len(pos)]
    objects["index_count"] = [3, 3, 120, 24]
    objects["attr_offset"][:, 0] = 0
    batches, regions = build_tables([1, 1, 40, 8])
    return Scene(objects, mesh, batches, regions), end, stale


def pingpong_frames(seed=15):
    """Three frames over one mesh whose invocation totals grow and then shrink, so that the culling buffers are reallocated between
    frames and the input partition is the copy the resize made.  Every object that was in the previous frame gets its previous first
    invocation (in range), the others NO_PREVIOUS; the order is shuffled between frames.  Returns (scene of every object, tables per
    frame)."""
    rng = np.random.default_rng(seed)
    sizes = [1, 31, 33, 255, 257, 700, 1500, 4097]
    counts = [sizes[i % len(sizes)] for i in range(160)]
    s = structural_scene(counts, seed, [i % 4 for i in range(160)], [(i // 3) % 4 for i in range(160)])
    members = [list(range(50)), list(range(120)), list(range(100, 160))]
    frames, prev_first = [], {}
    for m in members:
        order = list(rng.permutation(m))
        prev = [prev_first.get(i, NO_PREVIOUS) for i in range(160)]
        b, r = build_tables(counts, prev=prev, order=order)
        frames.append((b, r))
        prev_first = {int(i["object_id"]): int(bb["batch_base_invocation"]) + int(i["invocation_start"]) for bb in b
                      for i in bb["object_culling_information"][:int(bb["total_objects"])]}
    return s, frames


HIGH_ID = 1 << 24


def high_vertex_id_scene():
    """Vertex ids of 2^24 and above whose positions lie inside the mesh buffer (3 x (2^24 + 8) words, about 201 MB).  The position fetch
    must use the whole 32-bit id, the packed index only its low 24 bits.  The low ids 0-5 hold a back-facing copy of the triangles,
    so a fetch through the masked id decides differently.  Objects 0 and 1 are atomic, object 2 non-atomic (its in-place slots)."""
    n_words = 3 * (HIGH_ID + 8)
    mesh = np.zeros(n_words, np.uint32)
    front = np.array([[(10, 10, 0.5), (50, 10, 0.5), (10, 50, 0.5)], [(100, 100, 0.5), (140, 100, 0.5), (100, 140, 0.5)]], F32)
    back = front[:, [0, 2, 1]]
    mesh[3 * HIGH_ID:3 * HIGH_ID + 18] = front.reshape(-1).view(np.uint32)
    idx_at = 64
    mesh[:18] = back.reshape(-1).view(np.uint32)                          # ids 0-5: the back-facing copy
    mesh[idx_at:idx_at + 6] = HIGH_ID + np.arange(6, dtype=np.uint32)
    objects = object_records(3)                              # object 2 non-atomic: batch-local 2 << 24 does not hide bit 24 of an id
    objects["first_index"] = [idx_at, idx_at, idx_at + 3]
    objects["index_count"] = 3
    batches, regions = build_tables([1, 1, 1], atomic=[1, 1, 0], keys=[0, 0, 2])
    return Scene(objects, mesh, batches, regions)


def hiz_sizes():
    return [(1920, 1080), (3840, 2160), (40, 24), (36, 36), (34, 34), (480, 270), (481, 270), (1, 777), (777, 1), (2, 2048), (4096, 2),
            (1, 1)]


HIZ_CASES = [(w, h, 1) for w, h in hiz_sizes()] + [(1920, 1080, 4), (481, 270, 4)]


FUSED = {(1920, 1080): 3, (3840, 2160): 3, (40, 24): 3, (36, 36): 2, (34, 34): 1, (480, 270): 1, (481, 270): 0}


def hiz_content(w, h, seed):
    """Occluders for the hi-Z size tests: a far background over all but the top-left quarter and the last row and column (the uncovered
    pixels read 0), random triangles in front of it, and one-pixel quads along the whole last row and column at depths below the
    background's.  With odd sizes the unique minimum of a footprint then sits in its extra row or column.  Reverse-Z: the larger depth
    is the nearer, and the pyramid keeps the smaller.  Returns (triangles in pixels, depth per triangle)."""
    rng = np.random.default_rng(seed)
    tris, z = [], []
    x0, y0 = w // 4, h // 4
    tris += [((x0, y0), (w - 1, y0), (w - 1, h - 1)), ((x0, y0), (w - 1, h - 1), (x0, h - 1))]
    z += [0.45, 0.45]
    for _ in range(40):
        c = rng.uniform(0, 1, 2) * (w - 1, h - 1)
        t = np.clip(np.round((c + rng.uniform(-0.3, 0.3, (3, 2)) * (w, h)) * 4) / 4, 0, (w - 1, h - 1))
        tris.append(tuple(map(tuple, t)))
        z.append(float(rng.uniform(0.5, 0.9)))
    for x in range(w):
        tris += [((x, h - 1), (x + 1, h - 1), (x + 1, h)), ((x, h - 1), (x + 1, h), (x, h))]
        z += [0.05 + 0.35 * rng.random()] * 2
    for y in range(h - 1):
        tris += [((w - 1, y), (w, y), (w, y + 1)), ((w - 1, y), (w, y + 1), (w - 1, y + 1))]
        z += [0.05 + 0.35 * rng.random()] * 2
    return tris, np.array(z, F32)


def render_hiz(backend, w, h, samples, seed=0):
    tris, z = hiz_content(w, h, seed)
    r = raster_scenes.build(backend, w, h, tris, z)
    raster_scenes.draw(r, w, h, samples)
    launches = backend.launch_count()
    backend.hiz_build()
    launches = backend.launch_count() - launches
    levels = read_pyramid(backend, len(ref.hiz_dims(w, h)))
    # level 0 is the min over the samples (resolve_depth_min.wgsl:18-27), which is what the depth resolve keeps as well
    depth = backend.readback_depth()
    assert np.array_equal(levels[0].view(np.uint32), depth.view(np.uint32)), f"{w}x{h}x{samples}: level 0 is not the resolved depth"
    backend.last_hiz_launches = launches
    return levels


def assert_pyramid(levels, w, h, what):
    want = ref.hiz_pyramid(levels[0])
    assert [l.shape[::-1] for l in levels] == ref.hiz_dims(w, h), f"{what}: level sizes"
    for m in range(1, len(levels)):
        bad = levels[m].view(np.uint32) != want[m].view(np.uint32)
        assert not bad.any(), f"{what}: level {m} differs from hi_z.wgsl at {np.count_nonzero(bad)} texels, first {np.argwhere(bad)[0]}"


def exact_runs(backend, samples):
    """The exact decision scene under every flag combination and a shadow camera: yields (what, got, want, header)."""
    pyramid = draw_occluders(backend, samples)
    tris, z, labels = exact_decision_triangles()
    s = triangle_scene(tris, z)
    upload(backend, s)
    n = len(s.objects)
    for flags in EXACT_FLAGS:
        for cam in (CAMERA_VIEWPORT, 0):
            hdr = ortho_header(256, 256, flags, n, shadow_index=cam)
            got = run_cull(backend, s, hdr, cam)
            want = reference_for(got, s, hdr, pyramid if cam == CAMERA_VIEWPORT else None)
            yield f"flags {flags} camera {cam:#x}", s, got, want, labels, pyramid


def check_exact(what, s, got, want, labels):
    # the f32 path is exact here: float64 decides every triangle the same way
    diff = np.nonzero(want["pass32"] != want["pass64"])[0]
    assert not len(diff), f"{what}: f32 and float64 differ on {[labels[i] for i in diff[:5]]}"
    assert_matches(got, want, s, what)


def perspective_runs(backend):
    tris, labels, proj = perspective_scene()
    s = world_triangle_scene(tris)
    backend.set_render_target(64, 64, 1, (0, 0, 0, 0))
    backend.forward_begin()
    backend.hiz_build()                                   # an empty depth buffer: a uniform pyramid of 0.0
    pyramid = read_pyramid(backend, len(ref.hiz_dims(64, 64)))
    upload(backend, s)
    for flags in (0, PCU_POSITIVE_AREA_VISIBLE, PCU_MULTISAMPLED):
        hdr = ortho_header(64, 64, flags, len(s.objects), proj=proj)
        got = run_cull(backend, s, hdr)
        yield f"perspective flags {flags}", s, got, reference_for(got, s, hdr, pyramid), labels


def check_perspective(what, s, got, want, labels, margin_floor=1.0):
    """Decisions equal the f32 reference everywhere; float64 is checked where the margin allows.  Returns the excluded labels."""
    assert_matches(got, want, s, what)
    m = ref.decision_margin(want["q64"], want["stage64"], want["flags"], want["viewport"])
    near = m <= margin_floor
    bad = (want["pass32"] != want["pass64"]) & ~near
    assert not bad.any(), f"{what}: f32 and float64 differ beyond the margin on {[labels[i] for i in np.nonzero(bad)[0][:5]]}"
    unit = [i for i, l in enumerate(labels) if l == "unit w"]
    assert (want["q64"]["clip"][0][unit, 3] == 1).all(), "the unit-w triangles must have w == 1.0 exactly"
    return sorted(labels[i] for i in np.nonzero(near)[0])


def structural_runs(backend):
    """Yields (what, scene, got, want, census): the ragged scene over two frames (NO_PREVIOUS, then in range / past the partition),
    superblock-boundary scenes of 4 x 32768 + {-256, 0, 256} invocations, the mesh-end scene in a fresh context and again after a
    larger mesh left stale words behind the smaller one."""
    s = ragged_scene()
    upload(backend, s)
    n = len(s.objects)
    hdr = ortho_header(256, 256, 0, n)
    got = run_cull(backend, s, hdr)
    yield "ragged frame 0", s, got, reference_for(got, s, hdr, None)
    first = {}
    for b in s.batches:
        for info in b["object_culling_information"][:int(b["total_objects"])]:
            first[int(info["object_id"])] = int(b["batch_base_invocation"]) + int(info["invocation_start"])
    total = total_invocations(s.batches)
    prev = [NO_PREVIOUS if i % 3 == 0 else (first[i] if i % 3 == 1 else total + 4096 * 32 + i) for i in range(n)]
    counts = [int(c) // 3 for c in s.objects["index_count"]]
    atomic = [0 if i in (0, 1, 254, 255) else 1 for i in range(n)]
    keys = [2 if i in (0, 1, 254, 255) else 0 for i in range(n)]
    b2, r2 = build_tables(counts, atomic=atomic, keys=keys, prev=prev)
    s2 = Scene(s.objects, s.mesh, b2, r2)
    got = run_cull(backend, s2, hdr)
    yield "ragged frame 1", s2, got, reference_for(got, s2, hdr, None)
    for delta in (0, -256, 256):
        s = superblock_scene(delta)
        upload(backend, s)
        hdr = ortho_header(256, 256, PCU_POSITIVE_AREA_VISIBLE, len(s.objects))
        got = run_cull(backend, s, hdr)
        yield f"superblock {delta:+d}", s, got, reference_for(got, s, hdr, None)


def mesh_end_runs(make_backend):
    """The mesh-end scene in a fresh context, and again after a larger mesh buffer whose words past the smaller one's end are stale
    (the allocation is kept, so the bulk copy of the index runs reads them).  Closes the contexts it makes."""
    s, end, stale = mesh_end_scene()
    for with_stale in (False, True):
        b = make_backend()
        try:
            if with_stale:
                b.set_mesh_buffer(stale)
            upload(b, s)
            hdr = ortho_header(256, 256, PCU_MULTISAMPLED, len(s.objects))
            got = run_cull(b, s, hdr)
            yield f"mesh end stale={with_stale}", s, got, reference_for(got, s, hdr, None)
        finally:
            b.close()


def stale_triangles(s, stale, got, hdr):
    """The decisions of object 2's triangle 37 and object 3's first triangle when robust access is honoured, and when the stale words
    past mesh_words were read instead."""
    robust = reference_for(got, s, hdr, None)
    stale_view = Scene(s.objects, stale, s.batches, s.regions)
    wrong = reference_for(got, stale_view, hdr, None)
    picks = []
    for b in s.batches:
        for info in b["object_culling_information"][:int(b["total_objects"])]:
            g = int(b["batch_base_invocation"]) + int(info["invocation_start"])
            if int(info["object_id"]) == 2:
                picks.append(g + 37)
            if int(info["object_id"]) == 3:
                picks.append(g)
    return robust["stage"][picks], wrong["stage"][picks]


def pingpong_runs(backend):
    """The three frames of pingpong_frames, each compared as it comes (no second cull): yields (what, scene, got, want)."""
    s, frames = pingpong_frames()
    upload(backend, s)
    hdr = ortho_header(256, 256, 0, len(s.objects))
    for k, (b, r) in enumerate(frames):
        fs = Scene(s.objects, s.mesh, b, r)
        got = run_cull(backend, fs, hdr, settle=False)
        yield f"ping-pong frame {k}", fs, got, reference_for(got, fs, hdr, None)


def pingpong_census(frames):
    """The index buffer is reallocated for frame 1 (next_pow2 of its elements grows) and frame 1 and 2 read previous bits in range."""
    inv = [total_invocations(b) for b, _ in frames]
    pow2 = lambda v: 1 << (int(v) - 1).bit_length()
    assert inv[0] < inv[1] > inv[2] and pow2(3 * inv[1]) > pow2(3 * inv[0])
    for b, _ in frames[1:]:
        prev = [int(i["previous_global_invocation"]) for bb in b for i in bb["object_culling_information"][:int(bb["total_objects"])]]
        assert sum(p != NO_PREVIOUS for p in prev) >= 20


def high_id_run(backend):
    s = high_vertex_id_scene()
    upload(backend, s)
    hdr = ortho_header(256, 256, PCU_MULTISAMPLED, len(s.objects))
    got = run_cull(backend, s, hdr)
    return s, got, reference_for(got, s, hdr, None), hdr


def check_high_id(s, got, want, hdr, what):
    assert_matches(got, want, s, what)
    assert want["pass32"].all(), f"{what}: the triangles behind ids >= 2^24 face the camera"
    masked = s.mesh.copy()
    masked[64:70] &= 0xFFFFFF
    low = reference_for(got, Scene(s.objects, masked, s.batches, s.regions), hdr, None)
    assert not low["pass32"].any(), "fetching the positions through the masked ids must decide differently"
    assert want["idx_pred"][:6].tolist() == [0, 1, 2, (1 << 24) | 0, (1 << 24) | 1, (1 << 24) | 2]
    assert want["idx_resid"][3 * 512:3 * 512 + 3].tolist() == [(2 << 24) | 3, (2 << 24) | 4, (2 << 24) | 5]


def big_census(s, ends):
    """More than two passes of the persistent grid (4224 workgroups at 4 CTAs / SM, 5280 at 5), and the end-of-buffer objects lie in
    workgroups past the first pass, on both sides of the staging guard."""
    total = total_invocations(s.batches)
    assert total // 256 > 2 * WARP_STRIDE
    end = len(s.mesh)
    wgs = {}
    for b in s.batches:
        for info in b["object_culling_information"][:int(b["total_objects"])]:
            wgs[int(info["object_id"])] = (int(b["batch_base_invocation"]) + int(info["invocation_start"])) // 256
    assert min(wgs[o] for o in ends) > 132 * 5 * 8
    runs = [(int(s.objects[o]["first_index"]) & ~3) + 100 for o in ends]
    assert (end + 4) in runs and any(r > end + 4 for r in runs) and any(r < end + 4 for r in runs)


def batched_frame_runs(backend):
    """One whole frame of a small cube field through BaseRenderGraph (the batch tables from batch_objects, host- or device-built),
    then each camera's cull compared with the reference fed the tables, MVPs and pyramid that cull used."""
    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings, per_camera_header
    from rend3_b200.scenes import cube_field_scene
    res = (480, 270)
    ev = cube_field_scene(n_objects=1500, seed=5, resolution=res, n_point_lights=0, shadow_resolution=256, pull_back=12.0, extent=30.0)
    BaseRenderGraph(backend).add_to_graph(ev, res, 1, BaseRenderGraphSettings())
    pyramid = read_pyramid(backend, len(ref.hiz_dims(*res)))
    n = len(ev.object_buffer)
    cams = [(CAMERA_VIEWPORT, per_camera_header(ev.camera, CAMERA_VIEWPORT, res, 1, n), pyramid)]
    cams += [(i, per_camera_header(sh.camera, i, (sh.size, sh.size), 1, n), None) for i, sh in enumerate(ev.shadows)]
    for cam, hdr, pyr in cams:
        batches, regions = backend.readback_batches(cam)
        s = Scene(ev.object_buffer, np.asarray(ev.mesh_buffer, np.uint32), batches, regions)
        got = dict(words=backend.readback_culling_results(cam, 0), prev=backend.readback_culling_results(cam, 1),
                   dc_pred=backend.readback_draw_calls(cam, 0), dc_resid=backend.readback_draw_calls(cam, 1),
                   idx_pred=backend.readback_indices(cam, 0), idx_resid=backend.readback_indices(cam, 1),
                   mvps=backend.readback_object_matrices(cam, 0, n)["model_view_proj"].reshape(n, 16))
        yield f"frame camera {cam:#x}", s, got, reference_for(got, s, hdr, pyr)
