"""A reference for the per-triangle cull and the hi-Z pyramid, written from the shaders rather than from the oracle.

It restates cull.wgsl (execute_culling :264-324, textureSampleMin :243-262, cs_main :326-390 with the write helpers :84-141 and
get_previous_culling_result :152-160), hi_z.wgsl :18-33 and the host side of culler.rs (the draw-call clear :642 and the buffer
layout :88-125).  execute_culling is evaluated twice, vectorised over triangles:

  * in numpy float32, one IEEE operation at a time (numpy never contracts a * b + c), in WGSL source order;
  * in float64, which also yields a decision margin, so that near-ties can be named instead of hidden.

Where WGSL leaves a choice open, the project's stated choice is used (DESIGN.md, robust-access note, and the oracle's comments):
  C1  determinant(mat3x3) is the cofactor expansion along the first row, (p0.x t0 - p1.x t1) + p2.x t2 (oracle/r3_oracle.c:554);
  C2  min / max are IEEE minNum / maxNum: a NaN operand loses (np.fmin / np.fmax);
  C3  round() is ties-to-even (np.rint);
  C4  ceil(log2(max(e, 1))) is exact on the bit pattern: the exponent, plus one if any mantissa bit is set;
  C5  an out-of-range hi-Z mip clamps to the last level and texel coordinates clamp into the level.  A NaN coordinate takes the low
      texel 0 (max(NaN, 0) = 0) and the high texel res - 1 (min(NaN, res - 1) = res - 1).
"""
import math

import numpy as np

from rend3_b200.layouts import CAMERA_VIEWPORT, INVALID_VERTEX, NO_PREVIOUS, PCU_MULTISAMPLED, PCU_POSITIVE_AREA_VISIBLE

# the stage that decided a triangle
BACKFACE, PIXEL_CENTRE, OCCLUDED, PASS = 0, 1, 2, 3
STAGE_NAMES = ("back-face", "pixel centre", "occlusion", "pass")

# relative rounding allowance of the f32 evaluation used by the margins: each margin is (distance of the float64 value from its
# threshold) / (this bound times the magnitude of the terms).  A decision can only differ between f32 and float64 below margin 1.
ROUNDING = 2.0 ** -18


# ------------------------------------------------------------------ hi-Z
def hiz_dims(w, h):
    """Level count floor(log2(max(w, h))) + 1, level i of max(w >> i, 1) x max(h >> i, 1) (hi_z.rs:170-171)."""
    n = int(max(w, h)).bit_length()
    return [(max(w >> i, 1), max(h >> i, 1)) for i in range(n)]


def hiz_pyramid(depth):
    """hi_z.wgsl fs_main (:18-33) level after level: the min over the 2x2 footprint (starting from 1.0, :25), plus one column / row when
    the source size is odd (:23,26-27), texels outside the source skipped.  `depth` is level 0, (h, w) float32."""
    levels = [np.asarray(depth, dtype=np.float32)]
    h0, w0 = levels[0].shape
    for dw, dh in hiz_dims(w0, h0)[1:]:
        src = levels[-1]
        sh, sw = src.shape
        kx, ky = 2 + (sw & 1), 2 + (sh & 1)
        pad = np.ones((2 * dh + ky, 2 * dw + kx), dtype=np.float32)   # skipped texels count as the 1.0 start value
        pad[:sh, :sw] = src
        out = np.ones((dh, dw), dtype=np.float32)
        for dx in range(kx):
            for dy in range(ky):
                out = np.fmin(out, pad[dy:dy + 2 * dh:2, dx:dx + 2 * dw:2][:dh, :dw])
        levels.append(out)
    return levels


def hiz_fused_levels(w, h):
    """How many levels r3_hiz_build derives in its head kernel (r3_shade.cu:959): while the source level has even dimensions, at most
    three; then per level the downsample kernel while the level has more than 4096 texels, the tail kernel for the rest."""
    dims = hiz_dims(w, h)
    fused = 0
    while fused < 3 and fused + 1 < len(dims) and dims[fused][0] % 2 == 0 and dims[fused][1] % 2 == 0:
        fused += 1
    m = fused + 1
    down = 0
    while m < len(dims) and dims[m][0] * dims[m][1] > 4096:
        m, down = m + 1, down + 1
    return fused, down, m < len(dims)


def ceil_log2(x):
    """C4 on float32 values (cull.wgsl:314; max(e, 1) applied by the caller): exact on the bit pattern, 128 for inf / NaN."""
    x = np.asarray(x, dtype=np.float32)
    b = x.view(np.uint32).astype(np.int64)
    e, m = (b >> 23) & 0xFF, b & 0x7FFFFF
    r = np.where(e == 255, 128, e - 127 + (m != 0))
    return np.where(x > 1.0, r, 0).astype(np.int64)


def ceil_log2_f64(x):
    """C4 for float64 values: the exact ceil(log2(x)) of the float64 value."""
    x = np.asarray(x, dtype=np.float64)
    out = np.zeros(x.shape, dtype=np.int64)
    for i, v in np.ndenumerate(x):
        if not v > 1.0:
            continue
        if not math.isfinite(v):
            out[i] = 128
            continue
        m, e = math.frexp(v)          # v = m 2^e, 0.5 <= m < 1
        out[i] = e - 1 if m == 0.5 else e
    return out


def texture_sample_min(pyramid, u, v, mip, dtype=np.float32):
    """textureSampleMin (cull.wgsl:243-262) on a pyramid of numpy levels, vectorised, with C5.  Returns the min of the four texels
    (low / high x and y) of level `mip`."""
    u, v = np.asarray(u, dtype=dtype), np.asarray(v, dtype=dtype)
    mip = np.minimum(np.asarray(mip, dtype=np.int64), len(pyramid) - 1)
    out = np.zeros(u.shape, dtype=np.float32)
    for m in np.unique(mip):
        sel = mip == m
        t = pyramid[int(m)]
        rh, rw = dtype(t.shape[0]), dtype(t.shape[1])
        px, py = u[sel] * rw - dtype(0.5), v[sel] * rh - dtype(0.5)          # :247
        with np.errstate(invalid="ignore"):
            lx, ly = np.fmax(np.floor(px), dtype(0)), np.fmax(np.floor(py), dtype(0))          # :249
            hx, hy = np.fmin(np.ceil(px), rw - dtype(1)), np.fmin(np.ceil(py), rh - dtype(1))  # :250
            lx, ly = np.fmin(lx, rw - dtype(1)), np.fmin(ly, rh - dtype(1))     # C5
            hx, hy = np.fmax(hx, dtype(0)), np.fmax(hy, dtype(0))
        x0, y0, x1, y1 = (a.astype(np.int64) for a in (lx, ly, hx, hy))
        r = np.fmin(np.fmin(t[y0, x0], t[y0, x1]), np.fmin(t[y1, x0], t[y1, x1]))   # :257-260
        out[sel] = r
    return out


# ------------------------------------------------------------------ execute_culling
def clip_positions(mvp, pos, dtype):
    """model_view_proj * vec4(v, 1.0) (cull.wgsl:268-270): mvp (n, 16) column-major, pos (n, 3) -> (n, 4).  Component r accumulates
    ((m[r] x + m[4 + r] y) + m[8 + r] z) + m[12 + r]; the product with 1.0 is exact."""
    m, p = np.asarray(mvp).astype(dtype), np.asarray(pos).astype(dtype)
    return np.stack([((m[:, r] * p[:, 0] + m[:, 4 + r] * p[:, 1]) + m[:, 8 + r] * p[:, 2]) + m[:, 12 + r] for r in range(4)], axis=1)


def execute_culling(mvp, tris, flags, resolution, viewport, pyramid, dtype=np.float32):
    """cull.wgsl:264-324 for n triangles.  mvp (n, 16), tris (n, 3, 3) object-space positions, `flags` the PCU flags, `resolution`
    the camera's (w, h), `viewport` False for a shadow camera, `pyramid` the hi-Z levels (None or [] when there are none: the kernels
    then read 0.0).  Returns (passes, stage, q) with q a dict of the intermediate values."""
    d = dtype
    n = len(tris)
    tris = np.asarray(tris)
    with np.errstate(all="ignore"):
        p = [clip_positions(mvp, tris[:, k], d) for k in range(3)]
        (x0, y0, _, w0), (x1, y1, _, w1), (x2, y2, _, w2) = ([q[:, i] for i in range(4)] for q in p)
        t0, t1, t2 = y1 * w2 - y2 * w1, y0 * w2 - y2 * w0, y0 * w1 - y1 * w0
        det = (x0 * t0 - x1 * t1) + x2 * t2                                               # :272, C1
        positive = bool(flags & PCU_POSITIVE_AREA_VISIBLE)
        backface = (det <= 0) if positive else (det >= 0)                                 # :274-279
        ndc = [q[:, :3] / q[:, 3:4] for q in p]                                           # :281-283
        mn = np.fmin(ndc[0][:, :2], np.fmin(ndc[1][:, :2], ndc[2][:, :2]))                # :285, C2
        mx = np.fmax(ndc[0][:, :2], np.fmax(ndc[1][:, :2], ndc[2][:, :2]))
        half = np.asarray(resolution, dtype=d) / d(2)                                     # :288
        mins, maxs = (mn + d(1)) * half, (mx + d(1)) * half                               # :289-290
        if flags & PCU_MULTISAMPLED:
            misses = np.zeros(n, dtype=bool)
        else:
            misses = np.any(np.rint(mins) == np.rint(maxs), axis=1)                       # :292-298, C3
        mint, maxt = (mn + d(1)) / d(2), (mx + d(1)) / d(2)                               # :305-308
        mint[:, 1], maxt[:, 1] = d(1) - mint[:, 1], d(1) - maxt[:, 1]
        uv = (maxt + mint) / d(2)                                                         # :310
        edges = maxs - mins                                                               # :311
        longest = np.fmax(np.fmax(edges[:, 0], edges[:, 1]), d(1))                        # :313-314
        mip = ceil_log2(longest) if d == np.float32 else ceil_log2_f64(longest)
        depth = np.fmax(np.fmax(ndc[0][:, 2], ndc[1][:, 2]), ndc[2][:, 2])                # :316
        if viewport and pyramid:
            occl = texture_sample_min(pyramid, uv[:, 0], uv[:, 1], mip, d).astype(d)      # :317
        else:
            occl = np.zeros(n, dtype=d)
        occluded = depth < occl                                                           # :319
    stage = np.full(n, PASS, dtype=np.int8)
    if viewport:
        stage[occluded] = OCCLUDED
    stage[misses] = PIXEL_CENTRE
    stage[backface] = BACKFACE
    q = dict(det=det, mins=mins, maxs=maxs, uv=uv, mip=mip, depth=depth, occl=occl, ndc=ndc, clip=p, half=half)
    return stage == PASS, stage, q


def decision_margin(q64, stage64, flags, viewport):
    """How far each float64 decision is from flipping, in units of a bound on the f32 evaluation's rounding (ROUNDING times the
    magnitude of the terms): the minimum over the tests the triangle reached.  Below 1 the f32 evaluation may decide otherwise.
      det        |det| / (ROUNDING * sum over the cofactor products of |x_i| (|y_j w_k| + |y_k w_j|))
      centre     distance of min/max_screen from a rounding tie (k + 1/2) / (ROUNDING * (|screen| + half resolution))
      occlusion  |depth - occlusion_depth| / (ROUNDING * |depth|); the pyramid the perspective scenes use is uniform, so the texel and
                 mip choice cannot change occlusion_depth
    A non-finite value in the float64 evaluation gets margin 0 unless every path agrees it is NaN."""
    (x0, y0, _, w0), (x1, y1, _, w1), (x2, y2, _, w2) = ([q[:, i] for i in range(4)] for q in q64["clip"])
    with np.errstate(all="ignore"):
        s = (np.abs(x0) * (np.abs(y1 * w2) + np.abs(y2 * w1)) + np.abs(x1) * (np.abs(y0 * w2) + np.abs(y2 * w0))
             + np.abs(x2) * (np.abs(y0 * w1) + np.abs(y1 * w0)))
        m = np.abs(q64["det"]) / (ROUNDING * s)
        m = np.where(np.isnan(q64["det"]), np.inf, np.nan_to_num(m, nan=0.0, posinf=np.inf))
        if not flags & PCU_MULTISAMPLED:
            scr = np.concatenate([q64["mins"], q64["maxs"]], axis=1)
            tie = np.abs(scr - (np.floor(scr) + 0.5))
            mc = np.min(np.where(np.isnan(scr), np.inf, tie / (ROUNDING * (np.abs(scr) + np.max(q64["half"])))), axis=1)
            mc = np.where(np.isfinite(scr).all(axis=1) | np.isnan(scr).any(axis=1), mc, 0.0)
            m = np.where(stage64 >= PIXEL_CENTRE, np.fmin(m, mc), m)
        if viewport:
            dd = q64["depth"].astype(np.float64)
            mo = np.abs(dd - q64["occl"].astype(np.float64)) / (ROUNDING * np.abs(dd))
            mo = np.where(np.isnan(dd), np.inf, np.nan_to_num(mo, nan=0.0, posinf=np.inf))
            m = np.where(stage64 >= OCCLUDED, np.fmin(m, mo), m)
    return m


def f32_ulps(a, b):
    """Signed distance from b to a in float32 units in the last place (both finite)."""
    def key(x):
        i = np.asarray(x, dtype=np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return key(a) - key(b)


# ------------------------------------------------------------------ cs_main + culler.rs for one camera
def mesh_words_at(mesh, idx):
    """Robust access (DESIGN.md): a word at or past the mesh buffer's end reads 0."""
    idx = np.asarray(idx, dtype=np.int64)
    ok = idx < len(mesh)
    return np.where(ok, mesh[np.where(ok, idx, 0)], 0).astype(np.uint32)


def cull_lists(batches, regions, mesh, objects, mvps, header, pyramid, prev_bits):
    """cs_main (cull.wgsl:326-390) over every batch of one camera, plus the host side of culler.rs.

    batches / regions: BATCH_DTYPE / REGION_DTYPE tables; mesh: the mesh buffer's u32 words; objects: OBJECT_DTYPE records; mvps
    (n_objects, 16): the baked model_view_proj of every object; header: CAMERA_HEADER_DTYPE; pyramid: hi-Z levels (ignored for a
    shadow camera); prev_bits: the visibility words of the previous cull (the input partition), read as 0 past their end.

    Triangles are appended to a region's lists in ascending invocation order.  The shader appends with atomics (:63-67), so it fixes
    only the SET of triangles per region; ascending order is one legal outcome and the project's documented choice (DESIGN.md;
    r3_tri_cull.cu).  `same_sets` compares lists without the order.

    Returns a dict: words (visibility bits, one per invocation), dc_pred / dc_resid (INDIRECT_CALL_DTYPE per region), idx_pred /
    idx_resid (uint32, INVALID_VERTEX where undefined), pred_defined / resid_defined (bool masks of the defined index words), stage
    (per invocation, -1 for padding) and margin inputs (q64, stage64, flags, viewport, f32 / f64 decisions)."""
    from rend3_b200.layouts import INDIRECT_CALL_DTYPE

    flags, res = int(header["flags"]), tuple(float(r) for r in header["resolution"])
    viewport = int(header["shadow_index"]) == CAMERA_VIEWPORT
    total = int(sum(int(b["total_invocations"]) for b in batches))
    n_words = (total + 31) // 32
    # gather every real triangle of every object
    rows = []
    for b in batches:
        base = int(b["batch_base_invocation"])
        for o in range(int(b["total_objects"])):
            rows.append((base, o, b["object_culling_information"][o]))
    gi_parts, oi_parts, ob_parts, info_rows = [], [], [], []
    for base, o, info in rows:
        s, e = int(info["invocation_start"]), int(info["invocation_end"])
        gi_parts.append(base + np.arange(s, e, dtype=np.int64))
        oi_parts.append(np.arange(e - s, dtype=np.int64))
        ob_parts.append(np.full(e - s, len(info_rows), dtype=np.int64))
        info_rows.append((base, o, info))
    gi = np.concatenate(gi_parts) if gi_parts else np.zeros(0, np.int64)          # global invocation
    oinv = np.concatenate(oi_parts) if oi_parts else np.zeros(0, np.int64)        # object invocation
    row = np.concatenate(ob_parts) if ob_parts else np.zeros(0, np.int64)
    obj_id = np.array([int(r[2]["object_id"]) for r in info_rows], dtype=np.int64)
    first_index = objects["first_index"][obj_id].astype(np.int64)
    pos_off = (objects["attr_offset"][obj_id, 0] // 4).astype(np.int64)
    ib = first_index[row] + oinv * 3                                                # vertex_fetch (cull.wgsl:9-32)
    idx = np.stack([mesh_words_at(mesh, ib + k) for k in range(3)], axis=1)
    fp = pos_off[row][:, None] + idx.astype(np.int64) * 3
    pos = np.stack([mesh_words_at(mesh, fp + c) for c in range(3)], axis=2).view(np.float32)   # (n, 3 vertices, 3)
    mvp = np.asarray(mvps, dtype=np.float32).reshape(-1, 16)[obj_id[row]]
    pass32, stage32, _ = execute_culling(mvp, pos, flags, res, viewport, pyramid, np.float32)
    pass64, stage64, q64 = execute_culling(mvp, pos, flags, res, viewport, pyramid, np.float64)

    words = np.zeros(n_words, dtype=np.uint32)
    np.bitwise_or.at(words, gi[pass32] // 32, (np.uint32(1) << (gi[pass32] % 32).astype(np.uint32)))
    stage = np.full(total, -1, dtype=np.int8)
    stage[gi] = stage32

    n_reg = len(regions)
    dc_pred, dc_resid = np.zeros(n_reg, INDIRECT_CALL_DTYPE), np.zeros(n_reg, INDIRECT_CALL_DTYPE)
    idx_pred = np.full(3 * total, INVALID_VERTEX, dtype=np.uint32)
    idx_resid = np.full(3 * total, INVALID_VERTEX, dtype=np.uint32)
    pred_def, resid_def = np.zeros(3 * total, bool), np.zeros(3 * total, bool)
    prev = np.asarray(prev_bits, dtype=np.uint32)
    pred_count, resid_count = np.zeros(n_reg, np.int64), np.zeros(n_reg, np.int64)
    # objects in invocation order: the appends then come out in ascending invocation order
    order = sorted(range(len(info_rows)), key=lambda k: info_rows[k][0] + int(info_rows[k][2]["invocation_start"]))
    offsets = np.concatenate([[0], np.cumsum([int(r[2]["invocation_end"]) - int(r[2]["invocation_start"]) for r in info_rows])])
    for k in order:
        base, o, info = info_rows[k]
        r = int(info["region_id"])
        s, e = int(info["invocation_start"]), int(info["invocation_end"])
        padded = s + (e - s + 255) // 256 * 256
        sl = slice(offsets[k], offsets[k + 1])
        passes = pass32[sl]
        packed = (np.uint32(o) << np.uint32(24)) | (idx[sl] & np.uint32(0xFFFFFF))         # pack_batch_indices: o << 24 | index
        if int(info["local_region_id"]) == 0 and e > s:                                   # init_draw_calls (cull.wgsl:47-61)
            for dc in (dc_pred, dc_resid):
                dc[r]["instance_count"], dc[r]["base_index"] = 1, (base + s) * 3
        if int(info["atomic_capable"]) == 1:
            surv = packed[passes]
            g0 = base + int(info["base_region_invocation"]) + pred_count[r]            # :89-98
            idx_pred[3 * g0:3 * (g0 + len(surv))] = surv.reshape(-1)
            pred_def[3 * g0:3 * (g0 + len(surv))] = True
            pred_count[r] += len(surv)
            if viewport:
                pg = int(info["previous_global_invocation"])
                if pg == NO_PREVIOUS:                                                     # :152-160
                    was = np.zeros(e - s, dtype=bool)
                else:
                    pgi = np.arange(e - s, dtype=np.int64) + pg
                    w = mesh_words_at(prev, pgi // 32)
                    was = ((w >> (pgi % 32).astype(np.uint32)) & 1).astype(bool)
                rs = packed[passes & ~was]
                g1 = base + int(info["base_region_invocation"]) + resid_count[r]       # :106-115
                idx_resid[3 * g1:3 * (g1 + len(rs))] = rs.reshape(-1)
                resid_def[3 * g1:3 * (g1 + len(rs))] = True
                resid_count[r] += len(rs)
        else:                                                                             # :374-380, padding :343-347
            g = base + s
            slots = np.full((padded - s, 3), INVALID_VERTEX, dtype=np.uint32)
            slots[:e - s][passes] = packed[passes]
            idx_resid[3 * g:3 * (g + padded - s)] = slots.reshape(-1)
            resid_def[3 * g:3 * (g + padded - s)] = True
            resid_count[r] += padded - s
    dc_pred["vertex_count"], dc_resid["vertex_count"] = 3 * pred_count, 3 * resid_count
    return dict(words=words, dc_pred=dc_pred, dc_resid=dc_resid, idx_pred=idx_pred, idx_resid=idx_resid, pred_defined=pred_def,
                resid_defined=resid_def, stage=stage, pass32=pass32, pass64=pass64, stage64=stage64, q64=q64, flags=flags,
                viewport=viewport, invocations=gi)


def same_sets(want, idx_pred, idx_resid, regions_atomic):
    """Order-free comparison: per region and list, the same multiset of packed triangles.  Returns a list of the regions that differ."""
    bad = []
    for name, have, defined in (("pred", idx_pred, want["pred_defined"]), ("resid", idx_resid, want["resid_defined"])):
        dc = want["dc_pred" if name == "pred" else "dc_resid"]
        for r in range(len(dc)):
            b0, n = int(dc[r]["base_index"]), int(dc[r]["vertex_count"])
            w = want["idx_" + name][b0:b0 + n].reshape(-1, 3)
            h = np.asarray(have[b0:b0 + n]).reshape(-1, 3)
            if regions_atomic[r]:
                w, h = np.sort(w.view("u4,u4,u4").ravel()), np.sort(h.view("u4,u4,u4").ravel())
            if w.tobytes() != h.tobytes():
                bad.append((name, r))
    return bad
