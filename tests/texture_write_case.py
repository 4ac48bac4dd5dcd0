"""A numpy restatement of r3_write_texture_regions[_device] (include/rend3_b200.h), written from the header's rules: which regions are
valid, where their bytes land and what the blobs hold afterwards; plus the textures, worlds and random region sets the texture-write tests
use."""
import numpy as np

from rend3_b200.bc import BLOCK_FORMATS
from rend3_b200.layouts import (SKYBOX_FACE, TEXFMT_COUNT, TEXTURE_REGION_DTYPE, texfmt_element_bytes, texfmt_is_block,
                                texfmt_level_shape)
from rend3_b200.texformats import STORAGE
from rend3_b200.world import Texture

def level_bytes(fmt, width, height, level):
    _, _, cols, rows = texfmt_level_shape(fmt, width, height, level)
    return cols * rows * texfmt_element_bytes(fmt)


def sky_face_bytes(sky):
    w, f = int(sky["width"]), int(sky["format"])
    return sum(level_bytes(f, w, w, l) for l in range(int(sky["mip_count"])))


def target(texture, descs, sky):
    """(blob name, byte offset of the target's level 0, format, width, height, mip count), or None when the target does not exist."""
    texture = int(texture)
    if texture & 0x80000000:
        f = texture & 0x7FFFFFFF
        if sky is None or f >= 6:
            return None
        w = int(sky["width"])
        return "sky", int(sky["byte_offset"]) + f * sky_face_bytes(sky), int(sky["format"]), w, w, int(sky["mip_count"])
    if texture >= len(descs):
        return None
    d = descs[texture]
    return "table", int(d["byte_offset"]), int(d["format"]), int(d["width"]), int(d["height"]), int(d["mip_count"])


def plan(r, descs, sky, nbytes):
    """(blob, destination offset, destination pitch, source offset, source pitch, row bytes, rows) of a valid region, None otherwise."""
    t = target(r["texture"], descs, sky)
    if t is None:
        return None
    blob, base, fmt, width, height, mips = t
    level, x, y, w, h = (int(r[k]) for k in ("level", "x", "y", "width", "height"))
    src_offset, src_pitch = int(r["src_offset"]), int(r["src_pitch"])
    if int(r["_reserved"]) != 0 or level >= mips or w == 0 or h == 0:
        return None
    lw, lh, cols, rows_total = texfmt_level_shape(fmt, width, height, level)
    if x + w > lw or y + h > lh:
        return None
    elem = texfmt_element_bytes(fmt)
    if texfmt_is_block(fmt):
        if x % 4 or y % 4 or (w % 4 and x + w != lw) or (h % 4 and y + h != lh):
            return None
        ex, ey, ec, er = x // 4, y // 4, -(-w // 4), -(-h // 4)
    else:
        ex, ey, ec, er = x, y, w, h
    row_bytes = ec * elem
    if src_offset % elem or src_pitch % elem or src_pitch < row_bytes:
        return None
    if src_offset + (er - 1) * src_pitch + row_bytes > nbytes:
        return None
    offset = base + sum(level_bytes(fmt, width, height, l) for l in range(level))
    pitch = cols * elem
    return blob, offset + ey * pitch + ex * elem, pitch, src_offset, src_pitch, row_bytes, er


def apply(table, descs, sky, regions, texels, sky_blob=None):
    """(table blob, skybox blob, per-region validity) after the regions: valid ones applied in order, invalid ones dropped.  `sky` is the
    skybox's descriptor (None: no skybox), the source's size is len(texels)."""
    src = np.ascontiguousarray(texels).reshape(-1).view(np.uint8)
    nbytes = len(src)
    out = {"table": np.array(table, dtype=np.uint8, copy=True), "sky": None if sky_blob is None else np.array(sky_blob, dtype=np.uint8, copy=True)}
    valid = []
    for r in regions:
        p = plan(r, descs, sky, nbytes)
        valid.append(p is not None)
        if p is None:
            continue
        blob, dst, dpitch, so, spitch, row_bytes, rows = p
        for k in range(rows):
            out[blob][dst + k * dpitch: dst + k * dpitch + row_bytes] = src[so + k * spitch: so + k * spitch + row_bytes]
    return out["table"], out["sky"], np.array(valid, dtype=bool)


def units(regions, descs, sky, nbytes, seg=2048):
    """Work units (row segments of at most `seg` bytes) of the valid regions."""
    total = 0
    for r in regions:
        p = plan(r, descs, sky, nbytes)
        if p is not None:
            total += p[6] * -(-p[5] // seg)
    return total


# ------------------------------------------------------------------ textures of every format
_BC_NAMES = {}
for _name, (_plain, _srgb, _) in BLOCK_FORMATS.items():
    _BC_NAMES[_plain] = (_name, False)
    if _srgb is not None:
        _BC_NAMES[_srgb] = (_name, True)
_STORAGE_NAMES = {f: name for name, (f, _) in STORAGE.items()}


def texture_for(fmt, width, height, rng, mips="generated"):
    """A Texture stored in format `fmt` (0 .. 30) with random content, a full mip chain unless mips != "generated"."""
    rgba = rng.integers(0, 256, (height, width, 4), dtype=np.uint8)
    if fmt in (0, 1):
        return Texture(rgba, srgb=fmt == 1, mips=mips)
    if fmt == 2:
        return Texture(rng.standard_normal((height, width, 4)).astype(np.float32), mips=mips)
    if fmt in (3, 4):
        return Texture(rgba, channels=1 if fmt == 3 else 2, mips=mips)
    if fmt in _BC_NAMES:
        name, srgb = _BC_NAMES[fmt]
        n = 1 if mips != "generated" else max(width, height).bit_length()
        blocks = [rng.integers(0, 256, level_bytes(fmt, width, height, l), dtype=np.uint8) for l in range(n)]
        return Texture(rgba, srgb=srgb, block_format=name, block_levels=blocks)
    return Texture(rgba, storage=_STORAGE_NAMES[fmt], mips=mips)


SHAPES = [(1, 1), (37, 21), (6, 6), (8, 4)]   # 37 x 21 -> 18 x 10 -> ... -> 1 x 1; 6 x 6 -> 3 x 3 -> 1 x 1 (ragged BC tails)


def every_format_world(seed=0, extra=()):
    """A Renderer whose table holds each of the 31 formats in every shape of SHAPES (plus `extra` (format, w, h) textures)."""
    from rend3_b200.world import Renderer

    rng = np.random.default_rng(seed)
    r = Renderer()
    for fmt in range(TEXFMT_COUNT):
        for w, h in SHAPES:
            r.add_texture_2d(texture_for(fmt, w, h, rng))
    for fmt, w, h in extra:
        r.add_texture_2d(texture_for(fmt, w, h, rng))
    return r


def random_region(rng, fmt, width, height, mips, texture, max_elems=None):
    """One valid rectangle of a random level (texel coordinates), as (texture, level, x, y, w, h, element columns, element rows)."""
    level = int(rng.integers(0, mips))
    lw, lh, cols, rows = texfmt_level_shape(fmt, width, height, level)
    ec, er = int(rng.integers(1, cols + 1)), int(rng.integers(1, rows + 1))
    if max_elems is not None:
        ec, er = min(ec, max_elems), min(er, max_elems)
    ex, ey = int(rng.integers(0, cols - ec + 1)), int(rng.integers(0, rows - er + 1))
    if texfmt_is_block(fmt):
        x, y = 4 * ex, 4 * ey
        return texture, level, x, y, min(4 * ec, lw - x), min(4 * er, lh - y), ec, er
    return texture, level, ex, ey, ec, er, ec, er


def pack_regions(rects, fmts, rng, pitch_slack=True, offset_slack=True):
    """TEXTURE_REGION_DTYPE regions for rects (from random_region) with random source bytes, a random gap before each source and a random
    pitch above the row bytes (both multiples of the element size), and the source buffer."""
    regions = np.zeros(len(rects), dtype=TEXTURE_REGION_DTYPE)
    cursor = 0
    for k, (texture, level, x, y, w, h, ec, er) in enumerate(rects):
        elem = texfmt_element_bytes(fmts[k])
        cursor += elem * int(rng.integers(0, 3)) if offset_slack else 0
        cursor = -(-cursor // elem) * elem
        pitch = ec * elem + (elem * int(rng.integers(0, 3)) if pitch_slack else 0)
        regions[k] = (cursor, texture, level, x, y, w, h, pitch, 0)
        cursor += (er - 1) * pitch + ec * elem
    texels = rng.integers(0, 256, max(cursor, 1), dtype=np.uint8)[:cursor]
    return regions, texels


def disjoint_rects(rng, descs, sky, n, textures=None, faces=()):
    """n random valid rectangles over the listed textures (default: all) and skybox faces, no two of one level meeting: each is drawn
    inside its own cell of a grid laid over the level (cells of up to 8 x 8 elements), cells taken without replacement."""
    cells = []
    targets = [(int(i),) for i in (range(len(descs)) if textures is None else textures)] + [(SKYBOX_FACE(f),) for f in faces]
    for (t,) in targets:
        _, _, fmt, width, height, mips = target(t, descs, sky)
        for level in range(mips):
            _, _, cols, rows = texfmt_level_shape(fmt, width, height, level)
            for cy in range(0, rows, 8):
                for cx in range(0, cols, 8):
                    cells.append((t, fmt, width, height, level, cx, cy, min(8, cols - cx), min(8, rows - cy)))
    assert len(cells) >= n, (len(cells), n)
    out, fmts = [], []
    for i in rng.choice(len(cells), n, replace=False):
        t, fmt, width, height, level, cx, cy, cw, ch = cells[int(i)]
        lw, lh, _, _ = texfmt_level_shape(fmt, width, height, level)
        ec, er = int(rng.integers(1, cw + 1)), int(rng.integers(1, ch + 1))
        ex, ey = cx + int(rng.integers(0, cw - ec + 1)), cy + int(rng.integers(0, ch - er + 1))
        if texfmt_is_block(fmt):
            x, y = 4 * ex, 4 * ey
            out.append((t, level, x, y, min(4 * ec, lw - x), min(4 * er, lh - y), ec, er))
        else:
            out.append((t, level, ex, ey, ec, er, ec, er))
        fmts.append(fmt)
    return out, fmts


def whole_level_rects(descs, sky, pairs):
    """Whole-level rectangles for (texture, level) pairs."""
    out, fmts = [], []
    for t, level in pairs:
        _, _, fmt, width, height, _ = target(t, descs, sky)
        lw, lh, cols, rows = texfmt_level_shape(fmt, width, height, level)
        out.append((t, level, 0, 0, lw, lh, cols, rows))
        fmts.append(fmt)
    return out, fmts
