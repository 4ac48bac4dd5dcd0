"""The scenes of the reference's golden images (tests/golden/reference_goldens.npz, produced by tests/golden/make_reference_goldens.py)
and the criteria they are held to.  Each scene rebuilds one rend3-test case (rend3-test/tests/{simple,object,shadow,msaa}.rs) or
examples/src/cube through the TestRunner mirror and renders it with the backend `load()` returns.  The reference's own criterion is
nv-flip Mean(0.0) for the flat tests — i.e. identical images — so those are compared exactly here; the lit images are compared to
+-1 LSB (plane) or with the reference's looser thresholds restated as LSB budgets (shadow/cube, examples/cube).
"""
import os

import numpy as np

from rend3_b200 import glam
from rend3_b200.routines import BaseRenderGraphSettings
from rend3_b200.runner import TestRunner
from rend3_b200.world import LEFT, RIGHT, Camera, DirectionalLight, MeshBuilder, Object, PbrMaterial, PointLight

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_goldens.npz"))
IDENT = glam.identity()


def runner(load, handedness=LEFT):
    return TestRunner(load(), handedness)


def raw_camera(proj=IDENT, view=IDENT):
    return Camera(("raw", proj), view)


def assert_identical(img, name):
    gold = GOLD[name]
    diff = np.abs(img.astype(int) - gold.astype(int))
    assert diff.max() == 0, f"{name}: {np.count_nonzero(diff.max(axis=2))} pixels differ (max {diff.max()})"


def empty(load):
    r = runner(load)
    r.renderer.set_camera_data(raw_camera())
    assert_identical(r.render_frame(), "simple/empty")


def triangle(load, handedness, winding, visible):
    """simple.rs:30-86 — handedness x winding => visible / back-face culled."""
    r = runner(load, handedness)
    pos = [(0.5, -0.5, 0), (0, 0.5, 0), (-0.5, -0.5, 0)] if winding == "Ccw" else [(0.5, -0.5, 0), (-0.5, -0.5, 0), (0, 0.5, 0)]
    mesh = MeshBuilder.new(pos, LEFT if winding == "Cw" else RIGHT).build()
    mat = r.add_unlit_material((0.25, 0.5, 0.75, 1.0))
    r.renderer.add_object(Object(r.renderer.add_mesh(mesh), mat, IDENT))
    r.renderer.set_camera_data(raw_camera())
    assert_identical(r.render_frame(), "simple/triangle" if visible else "simple/triangle-backface")


COORD_TESTS = [
    ("NegZ", (1, 0, 0), (0, 1, 0), (0, 0, -1)),
    ("Z", (-1, 0, 0), (0, 1, 0), (0, 0, 1)),
    ("NegY", (1, 0, 0), (0, 0, -1), (0, -1, 0)),
    ("Y", (1, 0, 0), (0, 0, 1), (0, 1, 0)),
    ("NegX", (0, 0, -1), (0, 1, 0), (-1, 0, 0)),
    ("X", (0, 0, 1), (0, 1, 0), (1, 0, 0)),
]


def coordinate_space(load):
    """simple.rs:88-142 — six triangles, look_at_lh from each axis."""
    r = runner(load)
    for _name, right, up, cam in COORD_TESTS:
        right, up, cam = (np.array(v, dtype=np.float32) for v in (right, up, cam))
        pos = [0.5 * right - 0.5 * up, -0.5 * right - 0.5 * up, 0.0 * right + 0.5 * up]
        color = cam * -0.25 if (cam < 0).any() else cam
        mat = r.add_unlit_material((color[0], color[1], color[2], 1.0))
        r.renderer.add_object(Object(r.renderer.add_mesh(MeshBuilder.new(pos, LEFT).build()), mat, IDENT))
    for name, _right, up, cam in COORD_TESTS:
        r.renderer.set_camera_data(raw_camera(view=glam.look_at_lh(cam, (0, 0, 0), up)))
        assert_identical(r.render_frame(), f"simple/coordinate-space-{name}")


def sample_coverage(load, samples):
    """msaa.rs:46-88 for SampleCount::One and ::Four: 64x64 shrinking quads — pins pixel-centre / sample-pattern
    coverage, the top-left rule and cull.wgsl's misses-pixel-centre test (skipped when multisampled) bit for bit."""
    r = runner(load)
    mat = r.add_unlit_material((1, 1, 1, 1))
    base = glam.mul(glam.from_translation((0.5, 0.5, 0.0)), glam.from_scale((0.5, 0.5, 1.0)))
    for x in range(64):
        for y in range(64):
            sx = np.float32(1.0) - np.float32(x) / np.float32(63.0)
            sy = np.float32(1.0) - np.float32(y) / np.float32(63.0)
            t = glam.mul(glam.mul(glam.from_translation((x, y, 0.0)), glam.from_scale((sx, sy, 1.0))), base)
            r.plane(mat, t)
    r.renderer.set_camera_data(raw_camera(proj=glam.orthographic_lh(0.0, 64.0, 64.0, 0.0, 0.0, 1.0)))
    img = r.render_frame(samples=samples)
    if samples == 1:
        assert_identical(img, "msaa/sample-coverage-1")
    else:
        # the reference's own goldens disagree on how alpha = 2/4 encodes (sample-coverage-4.png stores 127, four.png 128:
        # they come from different drivers), so: identical per-pixel sample counts, identical RGB, alpha within 1 LSB
        gold = GOLD["msaa/sample-coverage-4"]
        assert np.array_equal(np.rint(img[..., 3] / 63.75), np.rint(gold[..., 3] / 63.75)), "per-pixel covered-sample counts differ"
        assert np.array_equal(img[..., :3], gold[..., :3])
        assert np.abs(img[..., 3].astype(int) - gold[..., 3].astype(int)).max() <= 1


def msaa_four(load):
    """msaa.rs:7-44 — the triangle at SampleCount::Four: 4x sample pattern, per-sample coverage, box resolve."""
    r = runner(load, LEFT)
    mesh = MeshBuilder.new([(0.5, -0.5, 0), (-0.5, -0.5, 0), (0, 0.5, 0)], LEFT).build()
    mat = r.add_unlit_material((0.25, 0.5, 0.75, 1.0))
    r.renderer.add_object(Object(r.renderer.add_mesh(mesh), mat, IDENT))
    r.renderer.set_camera_data(raw_camera())
    assert_identical(r.render_frame(samples=4), "msaa/four")


def multi_frame_add(load):
    """object.rs:67-109 — object buffer growth past STARTING_SIZE across two frames."""
    r = runner(load)
    mat = r.add_unlit_material((1, 1, 1, 1))
    base = glam.mul(glam.from_translation((0.5, 0.5, 0.0)), glam.from_scale((0.5, 1.0, 1.0)))
    r.renderer.set_camera_data(raw_camera(proj=glam.orthographic_lh(0.0, 2.0, 16.0, 0.0, 0.0, 1.0)))
    for x in range(2):
        for y in range(16):
            r.plane(mat, glam.mul(glam.from_translation((x, y, 0.0)), base))
        assert_identical(r.render_frame(), f"object/multi-frame-add-{x}")


def duplicate_object_retain(load):
    """object.rs:9-60 — a dropped object must not survive through the predicted pass."""
    r = runner(load)
    r.renderer.set_camera_data(raw_camera())
    mat = r.add_unlit_material((1, 1, 1, 1))
    t1 = glam.from_scale_rotation_translation((-0.25, 0.25, 0.25), glam.QUAT_IDENTITY, (-0.5, 0.0, 0.0))
    o1 = r.plane(mat, t1)
    assert_identical(r.render_frame(), "object/duplicate-object-retain-left")
    t2 = glam.from_scale_rotation_translation((-0.25, 0.25, 0.25), glam.QUAT_IDENTITY, (0.5, 0.0, 0.0))
    r.renderer.duplicate_object(o1, transform=t2)
    r.renderer.remove_object(o1)
    assert_identical(r.render_frame(), "object/duplicate-object-retain-right")


def shadow_scene(load):
    r = runner(load)
    r.add_directional_light((-1.0, -1.0, 1.0))
    m1 = r.add_lit_material((0.25, 0.5, 0.75, 1.0))
    r.plane(m1, glam.from_rotation_x(-np.float32(np.pi / 2)))
    r.renderer.set_camera_data(
        Camera(("orthographic", (2.5, 2.5, 5.0)), glam.look_at_lh((0.0, 1.0, -1.0), (0, 0, 0), (0, 1, 0)))
    )
    return r


def shadow_plane(load):
    """shadow.rs:9-35 — lit BRDF known answer: albedo/pi * n.l, no specular (a = 0), unshadowed."""
    r = shadow_scene(load)
    img = r.render_frame(size=256)
    gold = GOLD["shadow/plane"]
    diff = np.abs(img.astype(int) - gold.astype(int)).max(axis=2)
    # Expected linear colour albedo/pi/sqrt(3) = (0.045944, 0.091888, 0.137832) encodes to (60.50, 85.46, 103.8):
    # the golden's (61, 86, 104) has green 0.54 LSB high, inside the 0.6 LSB a hardware sRGB encoder is
    # allowed — so coverage must be identical and every channel within 1 LSB.
    assert np.array_equal(img[..., 3] > 0, gold[..., 3] > 0), "coverage differs"
    assert diff.max() <= 1, f"max LSB diff {diff.max()}, {np.count_nonzero(diff)} px differ"
    assert np.array_equal(img[..., 0], gold[..., 0]) and np.array_equal(img[..., 2], gold[..., 2])


def shadow_cube(load):
    """shadow.rs:37-53 — cube casting onto the plane (shadow map + PCF5 + self shadowing).  The reference
    accepts FLIP p50 <= 0.04; restated: the median pixel is identical and >= 97% are within 2 LSB."""
    r = shadow_scene(load)
    r.render_frame(size=256)
    m2 = r.add_lit_material((0.75, 0.5, 0.25, 1.0))
    r.cube(m2, glam.from_scale_rotation_translation((0.25, 0.25, 0.25), glam.QUAT_IDENTITY, (0.25, 0.25, -0.25)))
    img = r.render_frame(size=256)
    gold = GOLD["shadow/cube"]
    diff = np.abs(img.astype(int) - gold.astype(int)).max(axis=2)
    assert np.median(diff) == 0
    assert np.count_nonzero(diff <= 2) >= 0.97 * diff.size, f"{np.count_nonzero(diff > 2)} px off by > 2 LSB"


def cube_example_screenshot(load):
    """examples/src/cube/mod.rs:70-181 at 1280x720 (FLIP Mean(0.01) in the reference): perspective
    camera, 2048^2 shadow map, two point lights.  >= 99% of pixels within 2 LSB, mean abs diff < 0.5 LSB."""
    r = runner(load)
    mat = r.renderer.add_material(PbrMaterial(albedo_value=(0.5, 0.5, 0.5, 1.0)))
    r.cube(mat, IDENT)
    view = glam.mul(glam.from_euler_xyz(-0.55, 0.5, 0.0), glam.from_translation((-3.0, -3.0, 5.0)))
    r.renderer.set_camera_data(Camera(("perspective", 60.0, 0.1), view))
    r.renderer.add_directional_light(
        DirectionalLight(color=(1, 1, 1), intensity=1.0, direction=(-1.0, -4.0, 2.0), distance=400.0, resolution=2048)
    )
    for pos, col in [((0.1, 1.2, -1.5), (1, 0, 0)), ((1.5, 1.2, -0.1), (0, 1, 0))]:
        r.renderer.add_point_light(PointLight(position=pos, color=col, radius=2.0, intensity=4.0))
    img = r.render_frame(resolution=(1280, 720), settings=BaseRenderGraphSettings(clear_color=(0.10, 0.05, 0.10, 1.0)))
    gold = GOLD["examples/cube"]
    diff = np.abs(img[..., :3].astype(int) - gold[..., :3].astype(int)).max(axis=2)
    assert np.count_nonzero(diff <= 2) >= 0.99 * diff.size, f"{np.count_nonzero(diff > 2)} px off by > 2 LSB"
    assert diff.mean() < 0.5
