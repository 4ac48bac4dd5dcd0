"""Exact coverage reference for the rasteriser, in Python integers and float64 (no oracle code).

Restates the raster rules of oracle/r3_oracle_forward.inc as a specification:
  R4  a sample is covered when it lies inside all three edges of the triangle; a sample exactly on an edge belongs to the
      triangle only when that edge is a top edge (horizontal, interior below it in the y-down framebuffer) or a left edge
      (interior to its right).
  R7  with four samples the sample points sit at (-2, -6), (6, -2), (-6, 2), (2, 6) sixteenths of a pixel from the pixel centre.
Vertices are given as snapped 24.8 framebuffer coordinates (integers, 256 per pixel, y down); pixel (x, y) has its centre at
(256 x + 128, 256 y + 128).

`path_census` restates how rend3_b200/csrc/r3_raster.cu picks a raster path for each sub-triangle, so a test can assert that
its scene reaches the path it claims to test.  Every constant below cites the line of r3_raster.cu it restates: a change there
must show up here in review.
"""
import numpy as np

SUBPIXEL = 256
SAMPLE_DX = (-32, 96, -96, 32)          # r3_raster.cu:200 (c_sample_dx), rule R7
SAMPLE_DY = (-96, -32, 32, 96)          # r3_raster.cu:201 (c_sample_dy)
SMALL_AREA = 64                         # r3_raster.cu:29  inline when the pixel box covers at most this many pixels
MEDIUM_MAX = 32                         # r3_raster.cu:30  warp-cooperative up to this box size on both axes
BAND_ROWS = 16                          # r3_raster.cu:32  rows per band item
LARGE_CAP = 1 << 22                     # r3_raster.cu:33  queued large sub-triangles
BAND_CAP = 1 << 24                      # r3_raster.cu:34  queued band items
FITS32_REACH = 11585                    # r3_raster.cu:119 32-bit edge arithmetic up to this reach (sub-pixels)
GUARD = 64                              # r3_raster.cu:28  guard band, in multiples of w (rule R1)


def _as_tris(tris):
    t = np.asarray(tris, dtype=np.int64).reshape(-1, 3, 2)
    assert np.all(np.abs(t) < 2 ** 30), "coordinates past 2^30 sub-pixels: int64 edge products could overflow"
    return t


def signed_area(tris):
    """Twice the signed area in the y-down framebuffer; positive for the orientation the kernels rasterise."""
    t = _as_tris(tris)
    return (t[:, 1, 0] - t[:, 0, 0]) * (t[:, 2, 1] - t[:, 0, 1]) - (t[:, 2, 0] - t[:, 0, 0]) * (t[:, 1, 1] - t[:, 0, 1])


def orient(tris):
    """Swap the last two vertices of negatively oriented triangles (the kernels draw front faces in that orientation)."""
    t = _as_tris(tris).copy()
    neg = signed_area(t) < 0
    t[neg, 1], t[neg, 2] = t[neg, 2].copy(), t[neg, 1].copy()
    return t


def _inside(ax, ay, bx, by, sx, sy):
    """Sample (sx, sy) on the inner side of edge a -> b of a positively oriented triangle, or on it when the edge is top / left."""
    e = (bx - ax) * (sy - ay) - (by - ay) * (sx - ax)
    dx, dy = bx - ax, by - ay
    top_left = (dy < 0) or (dy == 0 and dx > 0)
    return (e > 0) | ((e == 0) & top_left)


def sample_offsets(samples):
    return ((0, 0),) if samples == 1 else tuple(zip(SAMPLE_DX, SAMPLE_DY))


def triangle_coverage(tri, width, height, samples):
    """Covered samples of one positively oriented triangle: (rows, cols, sample index) arrays, clipped to the target."""
    t = [[int(v) for v in p] for p in tri]
    xs, ys = [p[0] for p in t], [p[1] for p in t]
    # pixels whose centre lies within 128 sub-pixels of the box: any sample of them may be covered
    x0, x1 = max((min(xs) - 128) // SUBPIXEL - 1, 0), min((max(xs) + 128) // SUBPIXEL + 1, width - 1)
    y0, y1 = max((min(ys) - 128) // SUBPIXEL - 1, 0), min((max(ys) + 128) // SUBPIXEL + 1, height - 1)
    out = []
    if x0 > x1 or y0 > y1:
        return out
    py, px = np.mgrid[y0:y1 + 1, x0:x1 + 1].astype(np.int64)
    for k, (dx, dy) in enumerate(sample_offsets(samples)):
        sx, sy = px * SUBPIXEL + 128 + dx, py * SUBPIXEL + 128 + dy
        inside = np.ones(sx.shape, dtype=bool)
        for a, b in ((0, 1), (1, 2), (2, 0)):
            inside &= _inside(t[a][0], t[a][1], t[b][0], t[b][1], sx, sy)
        out.append((py[inside], px[inside], k))
    return out


def coverage(tris_24_8, width, height, samples, z=None):
    """Exact coverage of a list of triangles (snapped 24.8 vertices, either orientation; zero-area triangles cover nothing).

    Returns (count, owner): `count` is the number of covered (triangle, sample) pairs inside the target, the kernels'
    forward_stats()[1]; `owner[y, x, k]` is the index of the triangle that wins sample k of pixel (x, y) in the depth test,
    the largest `z` (later index on equal z), or -1 where no triangle covers the sample."""
    t = orient(tris_24_8)
    area = signed_area(t)
    z = np.zeros(len(t)) if z is None else np.asarray(z, dtype=np.float64)
    owner = np.full((height, width, samples), -1, dtype=np.int64)
    front = np.full((height, width, samples), -np.inf)
    count = 0
    for i in range(len(t)):
        if area[i] == 0:
            continue
        for ry, rx, k in triangle_coverage(t[i], width, height, samples):
            count += len(ry)
            win = z[i] >= front[ry, rx, k]
            owner[ry[win], rx[win], k] = i
            front[ry[win], rx[win], k] = z[i]
    return count, owner


def covered_count(tris_24_8, width, height, samples):
    """forward_stats()[1] of many triangles, evaluating each shape once: coverage does not change under a translation by whole
    pixels while the triangle stays inside the target, so triangles equal up to such a translation share one evaluation."""
    t = orient(tris_24_8)
    t = t[signed_area(t) != 0]
    lo, hi = t.min(axis=1), t.max(axis=1)
    inside = (lo[:, 0] >= 0) & (lo[:, 1] >= 0) & (hi[:, 0] < width * SUBPIXEL) & (hi[:, 1] < height * SUBPIXEL)
    total = 0
    for tri in t[~inside]:
        total += sum(len(ry) for ry, _, _ in triangle_coverage(tri, width, height, samples))
    base = (lo[inside] // SUBPIXEL) * SUBPIXEL
    shapes, counts = np.unique((t[inside] - base[:, None, :]).reshape(-1, 6), axis=0, return_counts=True)
    for shape, n in zip(shapes, counts):
        shape = shape.reshape(3, 2)
        box = (shape.max(axis=0) + 2 * SUBPIXEL) // SUBPIXEL + 2   # a target large enough to hold the shape unclipped
        total += int(n) * sum(len(ry) for ry, _, _ in triangle_coverage(shape + SUBPIXEL, int(box[0]) + 1, int(box[1]) + 1, samples))
    return total


def plane_depth(tri_24_8, z3, sx, sy):
    """Depth of the triangle's plane (rule R5 in exact arithmetic) at sample points (sx, sy) in sub-pixels, in float64."""
    t = orient([tri_24_8])[0].astype(np.float64)
    swapped = signed_area([tri_24_8])[0] < 0
    z3 = np.asarray(z3, dtype=np.float64)
    if swapped:
        z3 = z3[[0, 2, 1]]
    (ax, ay), (bx, by), (cx, cy) = t
    area = (bx - ax) * (cy - ay) - (cx - ax) * (by - ay)
    la = ((cx - bx) * (sy - by) - (cy - by) * (sx - bx)) / area
    lb = ((ax - cx) * (sy - cy) - (ay - cy) * (sx - cx)) / area
    lc = ((bx - ax) * (sy - ay) - (by - ay) * (sx - ax)) / area
    return np.clip(la * z3[0] + lb * z3[1] + lc * z3[2], 0.0, 1.0)


def f32_ulps(a, b):
    """Distance in f32 units in the last place between two arrays of non-negative floats."""
    return np.abs(np.asarray(a, np.float32).view(np.int32).astype(np.int64) - np.asarray(b, np.float32).view(np.int32).astype(np.int64))


def snap_exact(xy_pixels):
    """24.8 integers of framebuffer positions given in pixels; asserts that snapping is exact (every position a multiple of 1/256
    pixel and small enough that the f32 transform, divide and snap of an orthographic camera lose nothing)."""
    p = np.asarray(xy_pixels, dtype=np.float64) * SUBPIXEL
    q = np.rint(p)
    assert np.array_equal(p, q), "positions must be multiples of 1/256 pixel"
    assert np.all(np.abs(q) < 2 ** 23), "positions must stay within 2^15 pixels for the f32 path to be exact"
    return q.astype(np.int64)


def small_primitive_culled(tris_24_8):
    """cull.wgsl's test for single-sampled targets (the triangle cull, before the rasteriser): a triangle is dropped when its
    screen-space box rounds (half to even) to the same pixel edge on either axis."""
    t = np.asarray(tris_24_8, dtype=np.float64).reshape(-1, 3, 2) / SUBPIXEL
    lo, hi = np.rint(t.min(axis=1)), np.rint(t.max(axis=1))
    return (lo[:, 0] == hi[:, 0]) | (lo[:, 1] == hi[:, 1])


# ------------------------------------------------------------------ which path the kernels take
def pixel_bounds(tri, samples, rect):
    """r3_raster.cu:305-315: pixels whose centre (1 sample) or any sample (4 samples) the box may reach, clamped to rect = (x0, y0, x1, y1)."""
    xs, ys = [int(v[0]) for v in tri], [int(v[1]) for v in tri]
    if samples == 1:
        px0, px1 = (min(xs) - 128 + 255) >> 8, (max(xs) - 128) >> 8
        py0, py1 = (min(ys) - 128 + 255) >> 8, (max(ys) - 128) >> 8
    else:
        px0, px1, py0, py1 = min(xs) >> 8, max(xs) >> 8, min(ys) >> 8, max(ys) >> 8
    return max(px0, rect[0]), max(py0, rect[1]), min(px1, rect[2] - 1), min(py1, rect[3] - 1)


def fits32(tri, px0, py0, px1, py1):
    """r3_raster.cu:137-143: 32-bit edge arithmetic when every vertex and the box lie within FITS32_REACH of the first pixel centre."""
    ox, oy = px0 * 256 + 128, py0 * 256 + 128
    reach = max((px1 - px0) * 256 + 128, (py1 - py0) * 256 + 128)
    for x, y in tri:
        reach = max(reach, abs(int(x) - ox), abs(int(y) - oy))
    return reach <= FITS32_REACH and abs(px0) < (1 << 20) and abs(py0) < (1 << 20)


PATHS = ("outside", "inline_int", "inline_ll", "coop_int", "coop_ll", "band")


def raster_path(tri, samples, rect, clipped=False):
    """The path r3_raster.cu:373-403 gives one oriented sub-triangle while the queues have room."""
    px0, py0, px1, py1 = pixel_bounds(tri, samples, rect)
    if px0 > px1 or py0 > py1:
        return "outside"
    w, h = px1 - px0 + 1, py1 - py0 + 1
    suffix = "_int" if fits32(tri, px0, py0, px1, py1) else "_ll"
    if w * h <= SMALL_AREA:
        return "inline" + suffix
    if not clipped and w <= MEDIUM_MAX and h <= MEDIUM_MAX:   # clipped sub-triangles are never handed to the warp
        return "coop" + suffix
    return "band"


def band_items(tri, samples, rect):
    """r3_raster.cu:382: band items a large sub-triangle reserves."""
    _, py0, _, py1 = pixel_bounds(tri, samples, rect)
    return py1 // BAND_ROWS - py0 // BAND_ROWS + 1


def path_census(tris_24_8, samples, rect, clipped=None):
    """Per-path counts of the sub-triangles (snapped, any orientation; zero-area ones are dropped before the rasteriser),
    plus the large sub-triangles and band items requested.  `queue_full` says whether either queue overflows, i.e. whether the
    last row of the path table (the fallback to the set-up kernel) is reached; which ones fall back depends on the order in
    which the GPU serves the reservations."""
    t = orient(tris_24_8)
    keep = signed_area(t) != 0
    clipped = np.zeros(len(t), dtype=bool) if clipped is None else np.asarray(clipped, dtype=bool)
    per = []
    for tri, c, k in zip(t, clipped, keep):
        per.append(raster_path(tri, samples, rect, bool(c)) if k else "dropped")
    per = np.array(per)
    out = {p: int(np.count_nonzero(per == p)) for p in PATHS}
    out["large"] = out["band"]
    out["band_items"] = int(sum(band_items(tri, samples, rect) for tri, p in zip(t, per) if p == "band"))
    out["queue_full"] = out["large"] > LARGE_CAP or out["band_items"] > BAND_CAP
    out["per_triangle"] = per
    return out


def clip_to_guard_band(poly_pixels, width, height):
    """Rule R1 for an orthographic camera (w = 1), restated in framebuffer pixels: Sutherland-Hodgman against the guard band
    |ndc| <= 64, in float64.  Only used to predict raster paths of clipped geometry, for shapes chosen far from every threshold."""
    lo_x, hi_x = (1 - GUARD) * width / 2, (1 + GUARD) * width / 2
    lo_y, hi_y = (1 - GUARD) * height / 2, (1 + GUARD) * height / 2
    poly = [tuple(map(float, p)) for p in poly_pixels]
    for axis, bound, sign in ((0, lo_x, 1), (0, hi_x, -1), (1, lo_y, 1), (1, hi_y, -1)):
        out = []
        for i in range(len(poly)):
            a, b = poly[i], poly[(i + 1) % len(poly)]
            da, db = sign * (a[axis] - bound), sign * (b[axis] - bound)
            if da >= 0:
                out.append(a)
                if db < 0:
                    t = da / (da - db)
                    out.append((a[0] + t * (b[0] - a[0]), a[1] + t * (b[1] - a[1])))
            elif db >= 0:
                t = db / (db - da)
                out.append((b[0] + t * (a[0] - b[0]), b[1] + t * (a[1] - b[1])))
        poly = out
        if len(poly) < 3:
            return []
    return [np.rint(np.array([poly[0], poly[q], poly[q + 1]]) * SUBPIXEL).astype(np.int64) for q in range(1, len(poly) - 1)]
