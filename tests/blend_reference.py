"""Exact reference for the blend (transparent) routine, in numpy (no oracle code).

Restates the transparent pass of rend3_b200 as a specification, for unlit materials, whose shaded colour is the material's albedo
value, so that every step is a correctly rounded f32 or f16 operation numpy reproduces bit for bit:

  collect   r3_raster.cu:187 (r3_oracle_forward.inc:1156): a fragment of a key-2 (blend) triangle is kept for a sample when its depth
            bits are >= the opaque depth bits of that sample; each kept fragment takes one node of the fragment pool, whether or not
            it later passes the depth test between transparent layers.  Only the scissor rows are collected (r3_raster.cu:767).
  order     r3_shade.cu:677-688 (r3_oracle_forward.inc:1100-1103): fragments are applied in draw order — objects back to front as
            batch_objects orders key-2 objects, then mesh order inside an object.
  depth     r3_shade.cu:700-701 (r3_oracle_forward.inc:1156-1157): GreaterEqual against the running depth of the sample (the opaque
            depth, then the last transparent fragment that passed), with depth write.
  R5        r3_raster.cu:166-171: z = ((la * z0) + (lb * z1)) + (lc * z2) in f32, la = f32(edge value) * (1 / f32(area)), clamped
            to [0, 1]; a constant-z triangle is not always exactly at its z, so the reference evaluates R5 itself.
  R8        r3_shade.cu:703-705 (r3_oracle_forward.inc:1160-1162): rgb' = (src.rgb * src.a) + (dst.rgb * (1 - src.a)),
            a' = src.a + (dst.a * (1 - src.a)) in f32, rounded to f16 after every layer.
  resolve   r3_shade.cu:709-725, 576-612 (r3_oracle_forward.inc:1168-1183): one sample: the f16 result (the parity target holds the
            f16 value of a blended pixel, the unrounded shading result of the others).  Four samples: ((s0 + s1) + (s2 + s3)) * 0.25
            over the f16 samples, depth the minimum over the samples.
  blit      r3_shade.cu:857-876 (blit.wgsl fs_main_scene / fs_main_monitor).

Geometry is given as snapped 24.8 framebuffer coordinates (tests/raster_reference.py), every triangle positively oriented, with
the f32 depth of each vertex as the kernels see it (clip z with w = 1)."""
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import numpy as np

import raster_reference as ref

f32 = np.float32


def f16(x):
    """Round-to-nearest-even to half precision, back in f32."""
    return np.asarray(x, dtype=f32).astype(np.float16).astype(f32)


@dataclass
class Draw:
    """One object of unlit triangles: `tris` snapped 24.8 vertices (n, 3, 2), positively oriented; `z` the f32 vertex depths (n, 3)."""
    tris: np.ndarray
    z: np.ndarray
    colour: Tuple[float, float, float, float]


@dataclass
class Result:
    hdr16: np.ndarray        # (H, W, 4) f32 values of the rgba16f target
    hdr32: np.ndarray        # (H, W, 4) the f32 parity target
    depth: np.ndarray        # (H, W) f32 resolved depth
    blended: np.ndarray      # (H, W) bool: pixels with at least one blended sample
    n_blended: int           # forward_stats()[3]: blended (sample, fragment) pairs
    n_nodes: int             # fragment-pool nodes the collect takes
    samples_f16: np.ndarray = field(repr=False, default=None)   # (H, W, S, 4) per-sample colour target


def sample_points(ry, rx, k, samples):
    dx, dy = ref.sample_offsets(samples)[k]
    return rx.astype(np.int64) * ref.SUBPIXEL + 128 + dx, ry.astype(np.int64) * ref.SUBPIXEL + 128 + dy


def r5_depth(tri, z3, sx, sy):
    """Rule R5 at sample points (sx, sy) of a positively oriented snapped triangle, in f32 as the kernels evaluate it."""
    (ax, ay), (bx, by), (cx, cy) = [(int(p[0]), int(p[1])) for p in tri]

    def edge(x0, y0, x1, y1):
        return (x1 - x0) * (sy - y0) - (y1 - y0) * (sx - x0)

    area = (bx - ax) * (cy - ay) - (by - ay) * (cx - ax)
    assert area > 0, "triangles must be positively oriented"
    inv = f32(1.0) / f32(area)
    la = edge(bx, by, cx, cy).astype(f32) * inv
    lb = edge(cx, cy, ax, ay).astype(f32) * inv
    lc = edge(ax, ay, bx, by).astype(f32) * inv
    z0, z1, z2 = (f32(v) for v in z3)
    z = (la * z0 + lb * z1) + lc * z2
    return np.minimum(np.maximum(z, f32(0.0)), f32(1.0)).astype(f32)


def fragments(draws: List[Draw], width, height, samples):
    """Covered samples of every triangle of `draws`, in draw order: (ry, rx, k, depth bits, colour) per triangle and sample index."""
    for d in draws:
        for tri, z3 in zip(np.asarray(d.tris), np.asarray(d.z, dtype=f32)):
            for ry, rx, k in ref.triangle_coverage(tri, width, height, samples):
                if len(ry):
                    sx, sy = sample_points(ry, rx, k, samples)
                    yield ry, rx, k, r5_depth(tri, z3, sx, sy).view(np.uint32), d


def expected(width, height, samples, clear, opaque: List[Draw], layers: List[Draw], rows: Optional[Tuple[int, int]] = None):
    """The frame after the opaque resolve and the blend routine.  `opaque` are drawn first (no two may tie in depth: the owner of
    equal keys depends on record ids), `layers` are the transparent objects in draw order.  `rows` = the scissor band."""
    r0, r1 = rows if rows is not None else (0, height)
    S = samples
    zbits = np.zeros((height, width, S), dtype=np.uint32)                     # clear depth 0
    col = np.broadcast_to(np.asarray(clear, dtype=f32), (height, width, S, 4)).copy()
    for ry, rx, k, z, d in fragments(opaque, width, height, S):
        win = z >= zbits[ry, rx, k]
        zbits[ry[win], rx[win], k] = z[win]
        col[ry[win], rx[win], k] = np.asarray(d.colour, dtype=f32)
    opaque_z = zbits.copy()
    samp = f16(col)                                                           # the rgba16f (multisampled) colour target
    blended = np.zeros((height, width), dtype=bool)
    n_blended = n_nodes = 0
    for ry, rx, k, z, d in fragments(layers, width, height, S):
        band = (ry >= r0) & (ry < r1)
        ry, rx, z = ry[band], rx[band], z[band]
        kept = z >= opaque_z[ry, rx, k]                                       # collect (r3_raster.cu:187)
        n_nodes += int(np.count_nonzero(kept))
        ry, rx, z = ry[kept], rx[kept], z[kept]
        ok = z >= zbits[ry, rx, k]                                            # GreaterEqual (r3_shade.cu:700)
        ry, rx, z = ry[ok], rx[ok], z[ok]
        zbits[ry, rx, k] = z                                                  # depth write (:701)
        src = np.asarray(d.colour, dtype=f32)
        a = src[3]
        inv = f32(1.0) - a
        dst = samp[ry, rx, k]
        out = np.empty_like(dst)
        out[:, :3] = f16(src[:3] * a + dst[:, :3] * inv)                       # R8 (:703-705)
        out[:, 3] = f16(a + dst[:, 3] * inv)
        samp[ry, rx, k] = out
        blended[ry, rx] = True
        n_blended += len(ry)
    zf = zbits.view(f32)
    if S == 1:
        hdr32 = np.where(blended[..., None], samp[:, :, 0], col[:, :, 0])
        depth = zf[:, :, 0].copy()
    else:
        hdr32 = ((samp[:, :, 0] + samp[:, :, 1]) + (samp[:, :, 2] + samp[:, :, 3])) * f32(0.25)
        depth = np.minimum(f32(1.0), zf.min(axis=2))
    hdr32 = hdr32.astype(f32)
    return Result(f16(hdr32), hdr32, depth.astype(f32), blended, n_blended, n_nodes, samp)


# ------------------------------------------------------------------ blit.wgsl
SRGB_EXPONENT = float(f32(1.0 / 2.4))      # r3_shade.cu:870, the f32 constant 1.0f / 2.4f
MONITOR_EXPONENT = float(f32(0.4166))      # r3_shade.cu:871, fs_main_monitor's approximation
LINEAR_KNEE = float(f32(0.0031308))


def blit(hdr16, srgb_target):
    """blit.wgsl in float64 on the rgba16f values: (8-bit result, mask of channels whose e * 255 + 0.5 lies within 1e-4 of an integer,
    where an f32 evaluation may round either way)."""
    x = np.asarray(hdr16, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        if srgb_target:
            e = np.where(x <= LINEAR_KNEE, x * float(f32(12.92)), 1.055 * np.power(np.maximum(x, 0.0), SRGB_EXPONENT) - 0.055)
        else:
            e = np.where(x > LINEAR_KNEE, 1.055 * np.power(np.maximum(x, 0.0), MONITOR_EXPONENT) - 0.055, x * float(f32(12.92)))
    e[..., 3] = x[..., 3]
    e = np.clip(e, 0.0, 1.0)
    v = e * 255.0 + 0.5
    tie = np.abs(v - np.rint(v)) < 1e-4
    return np.floor(v).astype(np.int64), tie


def assert_blit(ldr, hdr16, srgb_target, what=""):
    want, tie = blit(hdr16, srgb_target)
    diff = np.abs(ldr.astype(np.int64) - want)
    bad = (diff > 1) | ((diff == 1) & ~tie)
    assert not bad.any(), f"{what}: {np.count_nonzero(bad)} 8-bit channels differ from blit.wgsl, first at {np.argwhere(bad)[0]}"
