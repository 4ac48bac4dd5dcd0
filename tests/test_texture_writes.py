"""Textures that change — r3_write_texture_regions, r3_write_texture_regions_device, r3_readback_texels — against the numpy restatement of
texture_write_case.py (blob bytes), r3_set_textures / r3_set_skybox of world.py's patched world (frames, bit for bit) and the CPU oracle
given that world, plus the calls' validation, the frame graph and the interplay with r3_update_textures / r3_set_textures."""
import ctypes
import os

import numpy as np
import pytest

import texture_write_case as twc
from harness import (ROOT, assert_same_frame, assert_same_ldr, check_declared_and_exported, expect_error, hdr_close, settings, to_device,
                     unbound_backend)
from rend3_b200.backend import R3Error, load_cuda_backend
from rend3_b200.layouts import SKYBOX_FACE, TEXTURE_REGION_DTYPE, texfmt_element_bytes, texfmt_is_block, texfmt_level_shape

E_INVALID, E_STATE = -1, -5


# ------------------------------------------------------------------ without a GPU
DECLS = ("int r3_write_texture_regions(r3_ctx*, const r3_texture_region* regions, uint32_t n, const void* texels, uint64_t nbytes);",
         "int r3_write_texture_regions_device(r3_ctx*, const r3_texture_region* d_regions, uint32_t n, const void* d_texels, uint64_t nbytes);",
         "int r3_readback_texels(r3_ctx*, int skybox, uint64_t byte_offset, void* out, uint64_t nbytes);")


def test_library_exports_the_three_entry_points_with_the_headers_signatures():
    check_declared_and_exported(DECLS, (None, None, ctypes.c_uint32(1), None, ctypes.c_uint64(0)))


def test_region_record_layout():
    layout = open(os.path.join(ROOT, "include", "r3_layouts.h")).read()
    assert 'R3_STATIC_ASSERT(sizeof(r3_texture_region) == 40, "r3_texture_region");' in layout
    assert "#define R3_SKYBOX_FACE(f) (0x80000000u | (f))" in layout
    want = {"src_offset": 0, "texture": 8, "level": 12, "x": 16, "y": 20, "width": 24, "height": 28, "src_pitch": 32, "_reserved": 36}
    for name, off in want.items():
        assert TEXTURE_REGION_DTYPE.fields[name][1] == off, name
        if name in ("texture", "level", "x", "width", "src_pitch", "_reserved"):
            assert f'R3_STATIC_ASSERT(offsetof(r3_texture_region, {name}) == {off}, "{name}");' in layout, name
    assert TEXTURE_REGION_DTYPE.itemsize == 40 and SKYBOX_FACE(5) == 0x80000005


def test_format_helpers_match_the_header_macros():
    """texfmt_element_bytes / texfmt_is_block against R3_TEXFMT_BPP / _BLOCK_BYTES / _IS_BLOCK, evaluated by a C compiler."""
    import subprocess
    import tempfile

    src = '#include <stdio.h>\n#include "r3_layouts.h"\nint main(void){for(unsigned f=0;f<R3_TEXFMT_COUNT;++f)' \
          'printf("%u %u\\n",(unsigned)R3_TEXFMT_IS_BLOCK(f),R3_TEXFMT_IS_BLOCK(f)?R3_TEXFMT_BLOCK_BYTES(f):R3_TEXFMT_BPP(f));return 0;}'
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "probe.c"), os.path.join(d, "probe")
        open(c, "w").write(src)
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        rows = [tuple(map(int, l.split())) for l in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split("\n") if l]
    assert rows == [(int(texfmt_is_block(f)), texfmt_element_bytes(f)) for f in range(31)]


@pytest.mark.parametrize("regions,texels", [
    (np.zeros(40, np.uint8), np.zeros(4, np.uint8)),                       # bytes, not records
    (np.zeros((2, 2), TEXTURE_REGION_DTYPE), np.zeros(4, np.uint8)),       # 2-d records
    (np.zeros(4, TEXTURE_REGION_DTYPE)[::2], np.zeros(4, np.uint8)),       # not contiguous
    (np.zeros(1, TEXTURE_REGION_DTYPE), np.zeros((4, 4), np.uint8)[:, :2]),  # texels not contiguous
    (np.zeros(1, TEXTURE_REGION_DTYPE), b"abcd"),                          # texels not an array
], ids=["bytes", "2d", "strided", "strided-texels", "bytes-object"])
def test_host_wrapper_rejects_bad_inputs_before_calling(regions, texels):
    with pytest.raises(AssertionError, match="regions|texels"):
        unbound_backend().write_texture_regions(regions, texels)


def test_device_wrapper_rejects_host_mistyped_and_misaligned_tensors_before_calling():
    torch = pytest.importorskip("torch")
    b = unbound_backend()
    good_host = torch.zeros(2, 40, dtype=torch.uint8)
    for regions, texels in ((good_host, good_host),                                         # host tensors
                            (np.zeros(2, TEXTURE_REGION_DTYPE), good_host),                 # a numpy array
                            (torch.zeros(2, 10, dtype=torch.float32), good_host),           # float rows
                            (torch.zeros(2, 41, dtype=torch.uint8), good_host),             # 41-byte rows
                            (torch.zeros(80, dtype=torch.uint8), good_host)):               # 1-d
        with pytest.raises(AssertionError):
            b.write_texture_regions_device(regions, texels)

    class FakeCuda:   # what the wrapper reads of a tensor, so that the checks run without a device
        def __init__(self, shape, esize, ptr, contiguous=True, floating=False):
            self.shape, self._e, self._p, self._c, self._f, self.is_cuda = shape, esize, ptr, contiguous, floating, True
        def dim(self): return len(self.shape)
        def element_size(self): return self._e
        def data_ptr(self): return self._p
        def is_contiguous(self): return self._c
        def is_floating_point(self): return self._f
        def numel(self): return int(np.prod(self.shape))
    tex = FakeCuda((64,), 1, 4096)
    for regions, n in ((FakeCuda((3, 40), 1, 4100), None),          # 4-byte aligned, not 8
                       (FakeCuda((3, 40), 1, 4096, contiguous=False), None),
                       (FakeCuda((3, 40), 1, 4096), 4),               # n past the rows
                       (FakeCuda((3, 40), 1, 4096), -1)):
        with pytest.raises(AssertionError):
            b.write_texture_regions_device(regions, tex, n)
    with pytest.raises(AssertionError):
        b.write_texture_regions_device(FakeCuda((3, 40), 1, 4096), FakeCuda((64,), 1, 4096, contiguous=False))


def _random_stored(rng, fmt, ec, er):
    return rng.integers(0, 256, (er, ec, texfmt_element_bytes(fmt)), dtype=np.uint8)


@pytest.mark.parametrize("fmt", range(31))
def test_world_writes_equal_the_restatement(fmt):
    """Renderer.write_texture_2d on textures of one format in the shapes 1x1, 37x21 (a full chain), 6x6 (BC tails 6x6, 3x3, 1x1) and 8x4:
    the next evaluate's blob equals the restatement applied to the previous blob with the emitted regions; every emitted region is valid;
    the levels not written keep their bytes (no regeneration); overlapping writes to one level go as one whole-level region."""
    from rend3_b200.world import Renderer

    rng = np.random.default_rng(100 + fmt)
    r = Renderer()
    for w, h in twc.SHAPES:
        r.add_texture_2d(twc.texture_for(fmt, w, h, rng))
    ev0 = r.evaluate()
    assert ev0.texture_writes is None
    descs = ev0.texture_descs
    for step in range(4):
        before = r.evaluate().texture_texels
        for _ in range(6):
            h = int(rng.integers(0, len(twc.SHAPES)))
            d = descs[h]
            t, level, x, y, w, hh, ec, er = twc.random_region(rng, fmt, int(d["width"]), int(d["height"]), int(d["mip_count"]), h)
            r.write_texture_2d(h, level, x, y, _random_stored(rng, fmt, ec, er))
        if step == 3:                                                   # the ragged tail of 37 x 21 and 6 x 6, whole
            for h, level in ((1, 5), (2, 1), (2, 2)):
                _, _, cols, rows = texfmt_level_shape(fmt, int(descs[h]["width"]), int(descs[h]["height"]), level)
                r.write_texture_2d(h, level, 0, 0, _random_stored(rng, fmt, cols, rows))
        ev = r.evaluate()
        regions, texels = ev.texture_writes
        got_table, _, valid = twc.apply(before, descs, None, regions, texels)
        assert valid.all(), f"step {step}: an emitted region is invalid"
        assert np.array_equal(got_table, ev.texture_texels), f"step {step}: the restatement differs from world.py's blob"
        for (a, b) in [(a, b) for i, a in enumerate(regions) for b in regions[:i]]:
            same = a["texture"] == b["texture"] and a["level"] == b["level"]
            meet = a["x"] < b["x"] + b["width"] and b["x"] < a["x"] + a["width"] and a["y"] < b["y"] + b["height"] and b["y"] < a["y"] + a["height"]
            assert not (same and meet), f"step {step}: emitted regions overlap"
    # a write to level 0 of a generated chain leaves level 1 as it was
    lv1_before = r.texture_levels[1][1].copy()
    r.write_texture_2d(1, 0, 0, 0, _random_stored(rng, fmt, 1, 1))
    assert np.array_equal(r.texture_levels[1][1], lv1_before)
    with pytest.raises(ValueError):
        r.write_texture_2d(1, 6, 0, 0, _random_stored(rng, fmt, 1, 1))           # level past the chain
    with pytest.raises(ValueError):
        r.write_texture_2d(0, 0, 0, 0, _random_stored(rng, fmt, 2, 1))           # past the 1x1 level
    with pytest.raises(ValueError):
        r.write_texture_2d(1, 0, 0, 0, np.zeros((1, 1, texfmt_element_bytes(fmt) + 1), np.uint8))
    if texfmt_is_block(fmt):
        with pytest.raises(ValueError):
            r.write_texture_2d(1, 0, 2, 0, _random_stored(rng, fmt, 1, 1))       # not on a block boundary


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
def test_world_skybox_writes_equal_the_restatement(dtype):
    from rend3_b200.world import Renderer

    rng = np.random.default_rng(7)
    r = Renderer()
    faces = [(rng.integers(0, 256, (8, 8, 4)) if dtype == np.uint8 else rng.standard_normal((8, 8, 4))).astype(dtype) for _ in range(6)]
    r.set_skybox(faces, srgb=True)
    ev0 = r.evaluate()
    for f in range(6):
        for level in (0, 1, 3):
            n = 8 >> level
            x, y = int(rng.integers(0, n)), int(rng.integers(0, n))
            patch = (rng.integers(0, 256, (n - y, n - x, 4)) if dtype == np.uint8 else rng.standard_normal((n - y, n - x, 4))).astype(dtype)
            r.write_skybox(f, level, x, y, patch)
    ev = r.evaluate()
    regions, texels = ev.texture_writes
    assert set(int(t) for t in regions["texture"]) == {SKYBOX_FACE(f) for f in range(6)}
    _, got_sky, valid = twc.apply(ev0.texture_texels, ev0.texture_descs, ev0.skybox_desc, regions, texels, ev0.skybox_texels)
    assert valid.all() and np.array_equal(got_sky, ev.skybox_texels)
    r.set_skybox(faces, srgb=True)                                        # new faces replace the writes
    ev2 = r.evaluate()
    assert ev2.texture_writes is None and np.array_equal(ev2.skybox_texels, ev0.skybox_texels)


# ------------------------------------------------------------------ GPU
def device_args(b, regions, texels):
    """(regions as uint8 (n, 40), texels as uint8) CUDA tensors made on the context's stream."""
    return to_device(b, np.ascontiguousarray(regions).view(np.uint8).reshape(-1, 40)), to_device(b, np.ascontiguousarray(texels).reshape(-1).view(np.uint8))


def blobs(b, table_len, sky_len):
    return b.readback_texels(False, 0, table_len), (b.readback_texels(True, 0, sky_len) if sky_len else None)


def sky_faces(rng, n, dtype):
    return [(rng.integers(0, 256, (n, n, 4)) if dtype == np.uint8 else rng.standard_normal((n, n, 4)) * 4.0).astype(dtype) for _ in range(6)]


@pytest.mark.gpu
def test_gpu_blob_bytes_equal_the_restatement():
    """Host- and device-form calls over every format (1x1 textures, 37x21 chains, 6x6 and 8x4 BC levels, a 512^2 R8 and a 1024^2 RGBA32F
    texture) and the six faces of an RGBA32F skybox: whole levels, ragged BC edges, odd R8 widths, 16-byte rows, source pitches above
    the row bytes, calls of 1, 33, 1000 and 5000 regions.  After each call the two blobs read back equal the restatement, byte for byte."""
    import torch

    from rend3_b200.layouts import TEXFMT_COUNT

    rng = np.random.default_rng(5)
    r = twc.every_format_world(seed=5, extra=[(3, 512, 512), (2, 1024, 1024)])
    r.set_skybox(sky_faces(rng, 32, np.float32), srgb=False)
    ev = r.evaluate()
    descs, sky = ev.texture_descs, ev.skybox_desc
    b = load_cuda_backend(0, parity_target=False)
    b.set_textures(descs, ev.texture_texels)
    b.set_skybox(sky, ev.skybox_texels)
    table, sky_blob = ev.texture_texels.copy(), ev.skybox_texels.copy()
    small = range(TEXFMT_COUNT * len(twc.SHAPES))
    big_r8, big_f32 = len(descs) - 2, len(descs) - 1
    every_level = [(t, l) for t in small for l in range(int(descs[t]["mip_count"]))]
    warps = torch.cuda.get_device_properties(0).multi_processor_count * 64
    calls = [
        ("every level of every small texture, whole", "host", *twc.whole_level_rects(descs, sky, every_level), True),
        ("the same, device", "device", *twc.whole_level_rects(descs, sky, every_level), True),
        ("one 1x1 region", "host", [(0, 0, 0, 0, 1, 1, 1, 1)], [0], True),
        ("33 regions, faces included", "device", *twc.disjoint_rects(rng, descs, sky, 33, faces=range(6)), True),
        ("1000 regions", "host", *twc.disjoint_rects(rng, descs, sky, 1000, faces=range(6)), True),
        ("1000 regions", "device", *twc.disjoint_rects(rng, descs, sky, 1000, faces=range(6)), True),
        ("5000 regions", "device", *twc.disjoint_rects(rng, descs, sky, 5000, faces=range(6)), True),
        ("5000 regions", "host", *twc.disjoint_rects(rng, descs, sky, 5000, faces=range(6)), False),
        ("16-byte rows: the 1024^2 RGBA32F level 0 and the faces' level 0", "device",
         *twc.whole_level_rects(descs, sky, [(big_f32, 0)] + [(SKYBOX_FACE(f), 0) for f in range(6)]), False),
        ("odd R8 widths", "host", [(big_r8, 0, 16 * k + 1, 9, w, 3, w, 3) for k, w in enumerate((1, 3, 7, 13))], [3] * 4, True),
    ]
    for label, form, rects, fmts, slack in calls:
        regions, texels = twc.pack_regions(rects, fmts, rng, pitch_slack=slack, offset_slack=slack)
        table, sky_blob, valid = twc.apply(table, descs, sky, regions, texels, sky_blob)
        assert valid.all(), label
        if len(regions) == 5000:
            assert twc.units(regions, descs, sky, len(texels)) > warps, f"{label}: fewer units than the grid has warps"
        if form == "host":
            b.write_texture_regions(regions, texels)
        else:
            d = device_args(b, regions, texels)
            b.write_texture_regions_device(*d)
        got_table, got_sky = blobs(b, len(table), len(sky_blob))
        assert np.array_equal(got_table, table), f"{label} ({form}): table blob"
        assert np.array_equal(got_sky, sky_blob), f"{label} ({form}): skybox blob"
    b.close()


def invalid_kinds(descs):
    """(label, region) for each way a region can be invalid, on a 37 x 21 BC7 texture (index BC7 * 4 + 1), a 37 x 21 RGBA32F texture
    (2 * 4 + 1) and a 37 x 21 R8 texture (3 * 4 + 1).  Source offsets count from the start of 4096 bytes that end the source."""
    bc7, f32, r8 = 15 * 4 + 1, 2 * 4 + 1, 3 * 4 + 1

    def reg(t, level, x, y, w, h, pitch, src_offset=0, reserved=0):
        r = np.zeros((), TEXTURE_REGION_DTYPE)
        r["src_offset"], r["texture"], r["level"], r["x"], r["y"], r["width"], r["height"], r["src_pitch"], r["_reserved"] = \
            src_offset, t, level, x, y, w, h, pitch, reserved
        return r
    return [
        ("texture past the table", reg(len(descs), 0, 0, 0, 1, 1, 16)),
        ("face 6", reg(SKYBOX_FACE(6), 0, 0, 0, 1, 1, 16)),
        ("level past the chain", reg(r8, 6, 0, 0, 1, 1, 1)),
        ("width 0", reg(r8, 0, 0, 0, 0, 1, 1)),
        ("height 0", reg(r8, 0, 0, 0, 1, 0, 1)),
        ("past the right edge", reg(r8, 0, 30, 0, 8, 1, 8)),
        ("past the bottom edge", reg(r8, 1, 0, 8, 1, 3, 1)),
        ("x + width wraps 32 bits", reg(r8, 0, 0xFFFFFFFF, 0, 2, 1, 2)),
        ("BC x not a multiple of 4", reg(bc7, 0, 2, 0, 4, 4, 16)),
        ("BC y not a multiple of 4", reg(bc7, 0, 0, 2, 4, 4, 16)),
        ("BC width ragged inside the level", reg(bc7, 0, 0, 0, 6, 4, 32)),
        ("BC height ragged inside the level", reg(bc7, 0, 0, 0, 4, 6, 16)),
        ("src_offset not a multiple of the element", reg(f32, 0, 0, 0, 2, 2, 32, src_offset=8)),
        ("src_pitch not a multiple of the element", reg(f32, 0, 0, 0, 1, 2, 24)),
        ("src_pitch below the row bytes", reg(f32, 0, 0, 0, 2, 2, 16)),
        ("last row past nbytes", reg(f32, 0, 0, 0, 2, 2, 32, src_offset=4096 - 48)),
        ("_reserved set", reg(r8, 0, 0, 0, 1, 1, 1, reserved=1)),
    ]


def with_invalid(regions, texels, bad, rng):
    """The valid regions with `bad` inserted at index 20, and their source: the valid texels, then 4096 bytes `bad` counts from."""
    base = -(-len(texels) // 16) * 16
    src = np.concatenate([texels, np.zeros(base - len(texels), np.uint8), rng.integers(0, 256, 4096, dtype=np.uint8)])
    bad = bad.copy()
    bad["src_offset"] += base
    return np.concatenate([regions[:20], bad.reshape(1), regions[20:]]), src


def valid_rects_apart(descs, sky, rng):
    """Valid regions on textures the invalid kinds do not touch (the 8 x 4 texture of every format) and on face 0."""
    targets = [fmt * 4 + 3 for fmt in range(31)]
    return twc.disjoint_rects(rng, descs, sky, 40, textures=targets, faces=(0,))


@pytest.mark.gpu
def test_gpu_device_form_drops_each_invalid_region_and_applies_the_others():
    rng = np.random.default_rng(9)
    r = twc.every_format_world(seed=9)
    r.set_skybox(sky_faces(rng, 8, np.uint8), srgb=True)
    ev = r.evaluate()
    descs, sky = ev.texture_descs, ev.skybox_desc
    b = load_cuda_backend(0, parity_target=False)
    b.set_textures(descs, ev.texture_texels)
    b.set_skybox(sky, ev.skybox_texels)
    table, sky_blob = ev.texture_texels.copy(), ev.skybox_texels.copy()
    keep = []
    for label, bad in invalid_kinds(descs):
        rects, fmts = valid_rects_apart(descs, sky, rng)
        regions, texels = twc.pack_regions(rects, fmts, rng)
        mixed, src = with_invalid(regions, texels, bad, rng)
        want_table, want_sky, valid = twc.apply(table, descs, sky, mixed, src, sky_blob)
        assert not valid[20] and valid[:20].all() and valid[21:].all(), label
        d = device_args(b, mixed, src)
        keep.append(d)
        b.write_texture_regions_device(*d)
        got_table, got_sky = blobs(b, len(table), len(sky_blob))
        assert np.array_equal(got_table, want_table) and np.array_equal(got_sky, want_sky), f"{label}: the drop differs"
        table, sky_blob = want_table, want_sky
    # faces without a skybox are dropped; a table alone is enough state
    nosky = load_cuda_backend(0, parity_target=False)
    nosky.set_textures(descs, ev.texture_texels)
    regions, texels = twc.pack_regions([(0, 0, 0, 0, 1, 1, 1, 1)], [0], rng)
    face = regions.copy()
    face["texture"] = SKYBOX_FACE(0)
    both = np.concatenate([regions, face])
    nosky.write_texture_regions_device(*device_args(nosky, both, texels))
    want, _, valid = twc.apply(ev.texture_texels, descs, None, both, texels)
    assert list(valid) == [True, False] and np.array_equal(nosky.readback_texels(False, 0, len(want)), want)
    nosky.close(), b.close()


@pytest.mark.gpu
def test_gpu_host_form_rejects_each_invalid_call_and_leaves_the_blobs():
    rng = np.random.default_rng(10)
    r = twc.every_format_world(seed=10)
    r.set_skybox(sky_faces(rng, 8, np.float32), srgb=False)
    ev = r.evaluate()
    descs, sky = ev.texture_descs, ev.skybox_desc
    b = load_cuda_backend(0, parity_target=False)
    b.set_textures(descs, ev.texture_texels)
    b.set_skybox(sky, ev.skybox_texels)
    before = blobs(b, len(ev.texture_texels), len(ev.skybox_texels))
    rects, fmts = valid_rects_apart(descs, sky, rng)
    regions, texels = twc.pack_regions(rects, fmts, rng)
    for label, bad in invalid_kinds(descs):
        mixed, src = with_invalid(regions, texels, bad, rng)
        with pytest.raises(R3Error) as e:
            b.write_texture_regions(mixed, src)
        assert e.value.code == E_INVALID, label
    over = np.concatenate([regions, regions[3:4]])                                     # a rectangle named twice
    expect_error(E_INVALID, b.write_texture_regions, over, texels)
    # two 4 x 4 rectangles of the 37 x 21 RGBA32F level 0 that share one texel; then ones that only touch
    corner, _ = twc.pack_regions([(9, 0, 0, 0, 4, 4, 4, 4), (9, 0, 3, 3, 4, 4, 4, 4)], [2, 2], rng)
    expect_error(E_INVALID, b.write_texture_regions, corner, np.zeros(1024, np.uint8))
    lib, ctx = b.lib, b.ctx
    assert lib.r3_write_texture_regions(ctx, None, ctypes.c_uint32(1), texels.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint64(len(texels))) == E_INVALID
    assert lib.r3_write_texture_regions(ctx, regions.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint32(len(regions)), None, ctypes.c_uint64(len(texels))) == E_INVALID
    assert lib.r3_write_texture_regions_device(ctx, None, ctypes.c_uint32(1), None, ctypes.c_uint64(0)) == E_INVALID
    got = blobs(b, len(ev.texture_texels), len(ev.skybox_texels))
    assert np.array_equal(got[0], before[0]) and np.array_equal(got[1], before[1]), "a rejected call wrote something"
    d = device_args(b, regions, texels)
    assert lib.r3_write_texture_regions_device(ctx, ctypes.c_void_p(d[0].data_ptr() + 4), ctypes.c_uint32(1), ctypes.c_void_p(d[1].data_ptr()),
                                               ctypes.c_uint64(len(texels))) == E_INVALID, "regions 4-byte aligned"
    b.write_texture_regions(regions[:0], texels)                                       # n == 0
    touch, _ = twc.pack_regions([(9, 0, 0, 0, 4, 4, 4, 4), (9, 0, 4, 0, 4, 4, 4, 4), (9, 0, 0, 4, 4, 4, 4, 4)], [2, 2, 2], rng)
    b.write_texture_regions(touch, np.zeros(1024, np.uint8))                           # edges that touch do not overlap
    expect_error(E_INVALID, b.readback_texels, False, len(ev.texture_texels) - 3, 4)
    expect_error(E_INVALID, b.readback_texels, True, 0, len(ev.skybox_texels) + 1)
    # R3_E_STATE without a table or a skybox; n == 0 is still R3_OK
    empty = load_cuda_backend(0, parity_target=False)
    expect_error(E_STATE, empty.write_texture_regions, regions, texels)
    expect_error(E_STATE, empty.write_texture_regions_device, *device_args(empty, regions, texels))
    empty.write_texture_regions(regions[:0], texels)
    empty.set_textures(descs[:0], np.zeros(0, np.uint8))
    expect_error(E_STATE, empty.write_texture_regions, regions, texels)
    empty.close(), b.close()


def quad_world(sample_type):
    from texture_case import build

    from rend3_b200.world import Texture

    rng = np.random.default_rng(3)
    r = build(None, Texture(rng.integers(0, 256, (64, 64, 4), dtype=np.uint8), srgb=True), sample_type=sample_type, uv_scale=1.5)
    return r.renderer, [0]


def cutout_world():
    from material_update_case import MaterialWorld

    w = MaterialWorld(n_objects=200)
    return w.r, w.textures


def scene_writes(r, handles, rng, frame):
    """One frame's edits: rectangles of level 0 and level 1 of every listed texture, and in the cutout world an alpha rewrite."""
    for h in handles:
        t = r.textures[h]
        n_levels = len(r.texture_levels[h]) if h in r.texture_levels else len(t.stored_levels())
        for level in range(min(2, n_levels)):
            lw, lh, _, _ = texfmt_level_shape(t.format(), t.data.shape[1], t.data.shape[0], level)
            w, hh = int(rng.integers(1, lw + 1)), int(rng.integers(1, lh + 1))
            x, y = int(rng.integers(0, lw - w + 1)), int(rng.integers(0, lh - hh + 1))
            patch = rng.integers(0, 256, (hh, w, 4), dtype=np.uint8)
            patch[..., 3] = np.where(rng.random((hh, w)) < 0.5, 20, 235) if frame % 2 else patch[..., 3]
            r.write_texture_2d(h, level, x, y, patch)


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["quad-nearest", "quad-linear", "cutout"])
@pytest.mark.parametrize("samples", [1, 4])
@pytest.mark.parametrize("form", ["host-eager", "device-graphed"])
def test_gpu_frames_equal_a_full_reupload_and_the_oracle(monkeypatch, scene, samples, form):
    """Five frames of texture writes (in the cutout world the albedo alpha of the per-fragment cutout material is rewritten, so the forward
    discard and the shadow pass's cutout change).  The writing context equals a context given r3_set_textures of world.py's patched table
    every frame in depth, rgba16f, the f32 parity target, LDR and the shadow atlas, bit for bit; the oracle given the same table agrees."""
    from oracle import load_oracle_backend
    from rend3_b200.backend import CAMERA_VIEWPORT
    from rend3_b200.routines import BaseRenderGraph

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    res = (96, 64)
    r, handles = cutout_world() if scene == "cutout" else quad_world(scene.split("-")[1])
    rng = np.random.default_rng(samples)
    ev = r.evaluate()
    wr, full, orc = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True), load_oracle_backend()
    gw, gf, go = BaseRenderGraph(wr), BaseRenderGraph(full), BaseRenderGraph(orc)
    for g in (gw, gf):
        g.add_to_graph(ev, res, samples, settings())
    keep = []
    for frame in range(5):
        scene_writes(r, handles, rng, frame)
        ev = r.evaluate()
        writes = ev.texture_writes
        if form == "device-graphed":
            keep.append(device_args(wr, *writes))
            writes = keep[-1]
        gw.add_to_graph(ev, res, samples, settings(), upload=False, frame_graph=form == "device-graphed", texture_writes=writes)
        full.set_textures(ev.texture_descs, ev.texture_texels)
        gf.add_to_graph(ev, res, samples, settings(), upload=False)
        what = f"{scene} frame {frame}"
        assert_same_frame(wr, full, ev, what)
        assert_same_ldr(wr, full, what)
        if ev.shadows:
            sw, sh = ev.shadow_target_size
            assert wr.readback_shadow_atlas(sw, sh).tobytes() == full.readback_shadow_atlas(sw, sh).tobytes(), f"{what}: atlas"
        go.add_to_graph(ev, res, samples, settings())
        assert np.array_equal(wr.readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32)), f"{what}: oracle depth"
        for cam in [CAMERA_VIEWPORT] + list(range(len(ev.shadows))):
            assert np.array_equal(wr.readback_visible(cam), orc.readback_visible(cam)), f"{what} camera {cam}: oracle"
        hdr_close(wr.readback_hdr_f32(), orc.readback_hdr_f32(), f"{what}: oracle hdr", scene == "cutout" or samples == 4)
    wr.close(), full.close(), orc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.uint8, np.float32], ids=["rgba8-srgb", "rgba32f"])
def test_gpu_skybox_writes_equal_set_skybox(dtype):
    """Writes into every face at levels 0, 1 and 3 (host form, then device form in a graph frame): the frame equals r3_set_skybox of
    world.py's patched faces, bit for bit, and the sky blob equals it byte for byte."""
    from rend3_b200.routines import BaseRenderGraph
    from rend3_b200.world import LEFT, Camera, Renderer
    from skybox_case import random_rotation

    rng = np.random.default_rng(4)
    res = (96, 64)
    r = Renderer(LEFT, aspect_ratio=res[0] / res[1])
    r.set_camera_data(Camera(("perspective", 90.0, 0.1), random_rotation(3)))
    r.set_skybox(sky_faces(rng, 16, dtype), srgb=dtype == np.uint8)
    ev = r.evaluate()
    wr, full = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    gw, gf = BaseRenderGraph(wr), BaseRenderGraph(full)
    for g in (gw, gf):
        g.add_to_graph(ev, res, 1, settings())
    keep = []
    for step, form in enumerate(("host", "device", "device")):
        for f in range(6):
            for level in (0, 1, 3):
                n = 16 >> level
                x, y = int(rng.integers(0, n)), int(rng.integers(0, n))
                w, h = int(rng.integers(1, n - x + 1)), int(rng.integers(1, n - y + 1))
                patch = (rng.integers(0, 256, (h, w, 4)) if dtype == np.uint8 else rng.standard_normal((h, w, 4)) * 8.0).astype(dtype)
                r.write_skybox(f, level, x, y, patch)
        ev = r.evaluate()
        writes = ev.texture_writes
        if form == "device":
            keep.append(device_args(wr, *writes))
            writes = keep[-1]
        gw.add_to_graph(ev, res, 1, settings(), upload=False, frame_graph=form == "device", texture_writes=writes)
        full.set_skybox(ev.skybox_desc, ev.skybox_texels)
        gf.add_to_graph(ev, res, 1, settings(), upload=False)
        assert np.array_equal(wr.readback_texels(True, 0, len(ev.skybox_texels)), ev.skybox_texels), f"step {step}: sky blob"
        assert_same_frame(wr, full, ev, f"step {step}")
        assert_same_ldr(wr, full, f"step {step}")
    wr.close(), full.close()


@pytest.mark.gpu
def test_gpu_graph_frames_stay_one_launch(monkeypatch):
    """Ten recorded frames of device-form writes whose count goes 1, 1000, 7, 1000, 500, ... with new contents each frame: once the plan
    scratch holds 1000 regions no frame flushes, every frame is graphed, the graphs are instantiated at most once per frame parity,
    and every frame equals a context given r3_set_textures of the patched table."""
    from material_update_case import MaterialWorld
    from rend3_b200.routines import BaseRenderGraph

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = MaterialWorld(n_objects=150, blend=False)   # a blend routine's fragment pool may grow (and flush) in any frame
    r = w.r
    big = r.add_texture_2d(twc.texture_for(0, 256, 256, np.random.default_rng(1)))
    ev = r.evaluate()
    res = (96, 64)
    wr, full = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    gw, gf = BaseRenderGraph(wr), BaseRenderGraph(full)
    for g in (gw, gf):
        g.add_to_graph(ev, res, 1, settings())
    rng = np.random.default_rng(2)
    table = ev.texture_texels.copy()
    descs = ev.texture_descs
    counts = [1000, 1, 1000, 7, 500, 1000, 1, 999, 250, 1000, 33]
    keep, first = [], None
    for frame, n in enumerate(counts):
        rects, fmts = twc.disjoint_rects(rng, descs, None, n, textures=[big] + list(w.textures))
        regions, texels = twc.pack_regions(rects, fmts, rng)
        table, _, _ = twc.apply(table, descs, None, regions, texels)
        d = device_args(wr, regions, texels)
        keep.append(d)
        gw.add_to_graph(ev, res, 1, settings(), upload=False, frame_graph=True, texture_writes=d)
        full.set_textures(descs, table)
        gf.add_to_graph(ev, res, 1, settings(), upload=False)
        assert_same_frame(wr, full, ev, f"frame {frame}")
        assert_same_ldr(wr, full, f"frame {frame}")
        if frame == 0:
            first = wr.frame_graph_stats()
    stats = wr.frame_graph_stats()
    print("frame graph stats", first, stats)
    assert stats["flushed"] == first["flushed"] and stats["graphed"] == first["graphed"] + len(counts) - 1, (first, stats)
    assert stats["instantiations"] - first["instantiations"] <= 2, (first, stats)
    wr.close(), full.close()


@pytest.mark.gpu
def test_gpu_writes_order_with_update_textures_and_set_textures():
    """r3_update_textures appends a texture past the blob's end (the blob grows), then a device write into it in the same frame lands in
    the grown blob; an r3_set_textures between two writes replaces everything, and a later write applies to the new table."""
    from rend3_b200.layouts import TEXTURE_DESC_DTYPE

    rng = np.random.default_rng(12)
    r = twc.every_format_world(seed=12)
    ev = r.evaluate()
    descs, table = ev.texture_descs, ev.texture_texels.copy()
    b = load_cuda_backend(0, parity_target=False)
    b.set_textures(descs, table)
    grown_tex = twc.texture_for(2, 64, 64, rng)
    lv = np.concatenate([np.ascontiguousarray(l).reshape(-1).view(np.uint8) for l in grown_tex.stored_levels()])
    off = len(table) + 4096 * 16
    nd = np.zeros(1, TEXTURE_DESC_DTYPE)
    nd[0] = (64, 64, len(grown_tex.stored_levels()), 2, off)
    b.frame_begin()
    b.update_textures(len(descs), nd, off, lv)
    descs2 = np.concatenate([descs, nd])
    table2 = np.concatenate([table, np.zeros(off - len(table), np.uint8), lv])
    rects, fmts = twc.disjoint_rects(rng, descs2, None, 50, textures=[len(descs), 0, 5])
    regions, texels = twc.pack_regions(rects, fmts, rng)
    d = device_args(b, regions, texels)
    b.write_texture_regions_device(*d)
    b.frame_end()
    want, _, valid = twc.apply(table2, descs2, None, regions, texels)
    assert valid.all() and np.array_equal(b.readback_texels(False, 0, len(want)), want), "write after the grown blob"
    # a set_textures between writes replaces everything; the next write applies to the new table
    b.set_textures(descs, ev.texture_texels)
    assert np.array_equal(b.readback_texels(False, 0, len(ev.texture_texels)), ev.texture_texels)
    expect_error(E_INVALID, b.readback_texels, False, 0, len(want))
    rects, fmts = twc.disjoint_rects(rng, descs, None, 40)
    regions, texels = twc.pack_regions(rects, fmts, rng)
    b.write_texture_regions(regions, texels)
    want, _, _ = twc.apply(ev.texture_texels, descs, None, regions, texels)
    assert np.array_equal(b.readback_texels(False, 0, len(want)), want)
    # a region naming the appended texture is past the replaced table: rejected by the host form, dropped by the device form
    late = twc.pack_regions([(len(descs), 0, 0, 0, 1, 1, 1, 1)], [2], rng)
    expect_error(E_INVALID, b.write_texture_regions, *late)
    b.write_texture_regions_device(*device_args(b, *late))
    assert np.array_equal(b.readback_texels(False, 0, len(want)), want)
    b.close()
