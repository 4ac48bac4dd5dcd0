"""Directional lights' shadow cameras evaluated on the device (rule R13, DESIGN.md §2): the numpy restatement
(shadow_camera_reference.py), the C oracle (oracle/r3_oracle_lights.c) and the CUDA kernel (r3_lights.cu) agree bit for bit, any NaN
equal to any NaN; the restatement stays close to world.shadow_camera (float64 inverse); frames driven through
add_to_graph(device_shadow_cameras=True) match the oracle and the host light path, stay one graph, and pass the reference's goldens."""
import numpy as np
import pytest

import shadow_camera_reference as ref
from harness import same_words_nan_equal
from oracle.lights import load_lights_oracle_backend
from reference_goldens import GOLD
from rend3_b200 import glam
from rend3_b200.backend import CAMERA_VIEWPORT, R3Error, load_cuda_backend
from rend3_b200.layouts import LIGHT_SOURCE_DTYPE, OBJECT_DTYPE
from rend3_b200.routines import BaseRenderGraphSettings
from rend3_b200.world import (CUTOUT, LEFT, RIGHT, Camera, CameraState, DirectionalLight, MeshBuilder, Object, PbrMaterial, Renderer,
                              Texture, shadow_camera)

f32 = np.float32
R3_E_INVALID, R3_E_STATE = -1, -5
ATLAS = (512, 256)


def random_sources(seed, n=6):
    rng = np.random.default_rng(seed)
    rows = [(tuple(rng.normal(size=3)), float(rng.uniform(0.5, 500.0)), int(rng.integers(16, 4096))) for _ in range(n)]
    s = ref.sources(rows)
    s["color"] = rng.random((n, 3))
    s["intensity"] = rng.uniform(0.0, 4.0, n)
    return s


# the edges R13 has to survive: a light along +-Y (a NaN camera), L on a texel boundary, negative coordinates (the sign of fmod),
# |L| around 1e6, a distance / resolution that is not a power of two, distance 0 (a NaN offset), a non-finite L
EDGE_SOURCES = ref.sources([((0.0, -1.0, 0.0), 40.0, 512), ((0.0, 1.0, 0.0), 40.0, 512), ((-1.0, -4.0, 2.0), 40.0, 512),
                        ((0.3, -0.8, -0.5), 10.0, 300), ((1.0, -1.0, 1.0), 0.0, 256), ((2.0, -3.0, -1.0), 400.0, 2048)])
EDGE_LOCATIONS = [(0.0, 0.0, 0.0), (1.5, 2.0, -3.0), (-7.25, -0.0390625, -13.5), (0.078125, 0.15625, 0.0), (-3.3, -17.9, -0.01),
                  (1.0e6, -3.0e5, 7.0), (-999999.9, 123456.7, -1.0e6), (np.inf, 0.0, 1.0), (np.nan, 1.0, 2.0)]


def cases():
    out = [("edges", EDGE_SOURCES, loc) for loc in EDGE_LOCATIONS]
    rng = np.random.default_rng(5)
    for seed in range(4):
        for _ in range(3):
            out.append((f"random{seed}", random_sources(seed), tuple(rng.uniform(-1e3, 1e3, 3) * 10.0 ** rng.integers(-3, 3))))
    return out


def evaluate(b, src, loc, left):
    b.set_directional_light_sources(src, ATLAS[0], ATLAS[1], left)
    b.evaluate_shadow_cameras(loc)
    return b.readback_shadow_cameras(len(src))


def check_equals_reference(b):
    for left in (True, False):
        for name, src, loc in cases():
            heads, lights = evaluate(b, src, loc, left)
            want_h, want_l = ref.evaluate(src, ATLAS[0], ATLAS[1], loc, left)
            assert same_words_nan_equal(heads, want_h), f"{name} {loc} left={left}: cameras differ"
            assert same_words_nan_equal(lights, want_l), f"{name} {loc} left={left}: light records differ"


def test_oracle_equals_numpy_r13_bit_for_bit():
    b = load_lights_oracle_backend()
    check_equals_reference(b)
    b.close()


def test_degenerate_cases_are_the_rules():
    """A light along +-Y has cross(Y, f) = 0: the whole camera is NaN.  distance 0 makes texel 0 and the offset NaN.  A non-finite L
    propagates.  A finite light and location give a finite camera."""
    for left in (True, False):
        h, _ = ref.evaluate(EDGE_SOURCES, ATLAS[0], ATLAS[1], (1.5, 2.0, -3.0), left)
        for i in (0, 1, 4):
            assert np.isnan(h[i]["view_proj"]).all() or np.isnan(h[i]["view_proj"]).sum() >= 12, i
        assert np.isfinite(h[2]["view_proj"]).all() and np.isfinite(h[3]["frustum"]).all()
        h, _ = ref.evaluate(EDGE_SOURCES, ATLAS[0], ATLAS[1], (np.inf, 0.0, 1.0), left)
        assert not np.isfinite(h[2]["view"]).all()


def test_texel_snapping_and_the_sign_of_fmod():
    """Moving the viewer within one texel leaves the camera's xy as it was; the offset keeps the dividend's sign, so a negative
    coordinate snaps towards zero like a positive one."""
    src = ref.sources([((0.0, 0.0, 1.0), 64.0, 64)])   # looking along +z: view xy = world xy (left-handed), texel = 1
    for x0, x1 in ((3.25, 3.75), (-3.25, -3.75)):
        a, _ = ref.evaluate(src, ATLAS[0], ATLAS[1], (x0, 0.5, 0.0), True)
        b, _ = ref.evaluate(src, ATLAS[0], ATLAS[1], (x1, 0.5, 0.0), True)
        assert same_words_nan_equal(a["view"], b["view"])
        assert a["view"][0][12] == -np.trunc(x0)


def world_camera(loc, left):
    return CameraState(Camera(("raw", glam.identity()), glam.from_translation(-np.asarray(loc, dtype=f32))), LEFT if left else RIGHT, None)


@pytest.mark.parametrize("left", [True, False])
def test_numpy_r13_is_close_to_world_shadow_camera(left):
    """world.shadow_camera inverts in float64; R13 in float32.  Bound: 2^-20 (1 + |L|) on every element of view, view_proj and the
    frustum planes (their normals are unit length, their distances grow with |L|)."""
    for seed in range(3):
        src = random_sources(seed)
        rng = np.random.default_rng(seed)
        for _ in range(4):
            loc = tuple(rng.uniform(-1e4, 1e4, 3))
            cam = world_camera(loc, left)
            assert np.allclose(cam.location(), loc, rtol=0, atol=1e-9 + 1e-7 * np.abs(loc).max())
            heads, _ = ref.evaluate(src, ATLAS[0], ATLAS[1], cam.location(), left)
            bound = 2.0 ** -20 * (1.0 + np.abs(cam.location()).max())
            for i, s in enumerate(src):
                light = DirectionalLight(tuple(s["color"]), float(s["intensity"]), tuple(s["direction"]), float(s["distance"]), int(s["resolution"]))
                w = shadow_camera(light, cam)
                assert np.abs(w.view.reshape(16) - heads[i]["view"]).max() <= bound
                assert np.abs(w.view_proj.reshape(16) - heads[i]["view_proj"]).max() <= bound
                assert np.abs(w.world_frustum - heads[i]["frustum"]).max() <= bound


def walkthrough_world(left, cutout=True, quad_roughness=0.6):
    """A ground plane, cubes, and a textured alpha-cutout quad that casts a shadow; a light straight down (-Y, a NaN camera) and a
    slanted one whose texel (20 / 256) the camera's steps cross."""
    from rend3_b200.runner import cube_mesh

    r = Renderer(LEFT if left else RIGHT, aspect_ratio=256 / 144)
    lit = r.add_material(PbrMaterial(albedo_value=(0.6, 0.5, 0.4, 1.0), roughness_factor=0.6))
    plane = MeshBuilder.new([(-1, 0, -1), (-1, 0, 1), (1, 0, 1), (1, 0, -1)], LEFT).with_indices([0, 1, 2, 0, 2, 3] if left else [0, 2, 1, 0, 3, 2]).build()
    r.add_object(Object(r.add_mesh(plane), lit, glam.from_scale((8.0, 1.0, 8.0))))
    cube = r.add_mesh(cube_mesh())
    for k in range(6):
        r.add_object(Object(cube, lit, glam.from_scale_rotation_translation((0.5, 0.5, 0.5), glam.QUAT_IDENTITY, (-3.0 + 1.2 * k, 0.5, 0.3 * k))))
    if cutout:
        data = np.full((16, 16, 4), 255, dtype=np.uint8)
        y, x = np.mgrid[0:16, 0:16]
        data[..., 3] = np.where(((x // 4) + (y // 4)) % 2 == 0, 230, 40)
        tex = r.add_texture_2d(Texture(data, srgb=False, mips="none"))
        # roughness > 0 by default: the -Y light grazes the vertical quad, where n.l is 0 up to rounding.  At roughness 0 a light with
        # n.l <= 0 makes surface_shading 0 * inf = NaN, which the final max() turns into the ambient term for the whole pixel, so the
        # sign of a rounding error in the normal decides whether the pixel is lit at all (test_gpu_walkthrough_roughness0_grazing_light)
        mat = r.add_material(PbrMaterial(albedo_texture=tex, albedo_value=(1.0, 1.0, 1.0, 1.0), transparency=CUTOUT, alpha_cutout=0.5, sample_type="nearest",
                                         roughness_factor=quad_roughness))
        quad = (MeshBuilder.new([(-1, -1, 0), (-1, 1, 0), (1, 1, 0), (1, -1, 0)], LEFT).with_indices([0, 2, 1, 0, 3, 2])
                .with_vertex_texture_coordinates_0([(0, 0), (0, 1), (1, 1), (1, 0)]).build())
        # double-sided: both windings, so the shadow pass (front faces culled) and the viewport each see one
        quad2 = (MeshBuilder.new([(-1, -1, 0), (-1, 1, 0), (1, 1, 0), (1, -1, 0)], LEFT).with_indices([0, 1, 2, 0, 2, 3])
                 .with_vertex_texture_coordinates_0([(0, 0), (0, 1), (1, 1), (1, 0)]).build())
        t = glam.from_scale_rotation_translation((1.5, 1.5, 1.0), glam.QUAT_IDENTITY, (0.5, 2.0, -1.0))
        r.add_object(Object(r.add_mesh(quad), mat, t))
        r.add_object(Object(r.add_mesh(quad2), mat, t))
    r.add_directional_light(DirectionalLight(color=(1.0, 1.0, 1.0), intensity=0.7, direction=(-1.0, -2.0, 0.5), distance=20.0, resolution=256))
    r.add_directional_light(DirectionalLight(color=(0.3, 0.3, 0.5), intensity=1.0, direction=(0.0, -1.0, 0.0), distance=20.0, resolution=128))
    return r


def walkthrough_camera(frame, left):
    eye = (0.5 + 0.047 * frame, 4.0 - 0.031 * frame, -9.0 + 0.061 * frame)
    view = (glam.look_at_lh if left else glam.look_at_rh)(eye, (0.0, 0.5, 0.0), (0.0, 1.0, 0.0))
    return Camera(("perspective", 60.0, 0.1), view)


def render_device(r, backend, resolution, settings=BaseRenderGraphSettings()):
    """TestRunner.render_frame with the shadow cameras evaluated on the device."""
    if resolution[0] != resolution[1]:
        r.renderer.set_aspect_ratio(resolution[0] / resolution[1])
    ev = r.renderer.evaluate()
    r.base_rendergraph.add_to_graph(ev, resolution, 1, settings, srgb_target=True, device_shadow_cameras=True)
    return backend.readback_ldr()


def check_goldens(make_backend):
    """tests/reference_goldens.py's shadow/cube and examples/cube criteria, with the cameras evaluated by R13."""
    from rend3_b200.runner import TestRunner
    from rend3_b200.world import PointLight

    b = make_backend()
    r = TestRunner(b, LEFT)
    r.add_directional_light((-1.0, -1.0, 1.0))
    r.plane(r.add_lit_material((0.25, 0.5, 0.75, 1.0)), glam.from_rotation_x(-np.float32(np.pi / 2)))
    r.renderer.set_camera_data(Camera(("orthographic", (2.5, 2.5, 5.0)), glam.look_at_lh((0.0, 1.0, -1.0), (0, 0, 0), (0, 1, 0))))
    render_device(r, b, (256, 256))
    r.cube(r.add_lit_material((0.75, 0.5, 0.25, 1.0)), glam.from_scale_rotation_translation((0.25, 0.25, 0.25), glam.QUAT_IDENTITY, (0.25, 0.25, -0.25)))
    img = render_device(r, b, (256, 256))
    diff = np.abs(img.astype(int) - GOLD["shadow/cube"].astype(int)).max(axis=2)
    assert np.median(diff) == 0
    assert np.count_nonzero(diff <= 2) >= 0.97 * diff.size, f"shadow/cube: {np.count_nonzero(diff > 2)} px off by > 2 LSB"
    b.close()
    b = make_backend()
    r = TestRunner(b, LEFT)
    r.cube(r.renderer.add_material(PbrMaterial(albedo_value=(0.5, 0.5, 0.5, 1.0))), glam.identity())
    r.renderer.set_camera_data(Camera(("perspective", 60.0, 0.1), glam.mul(glam.from_euler_xyz(-0.55, 0.5, 0.0), glam.from_translation((-3.0, -3.0, 5.0)))))
    r.renderer.add_directional_light(DirectionalLight(color=(1, 1, 1), intensity=1.0, direction=(-1.0, -4.0, 2.0), distance=400.0, resolution=2048))
    for pos, col in [((0.1, 1.2, -1.5), (1, 0, 0)), ((1.5, 1.2, -0.1), (0, 1, 0))]:
        r.renderer.add_point_light(PointLight(position=pos, color=col, radius=2.0, intensity=4.0))
    img = render_device(r, b, (1280, 720), BaseRenderGraphSettings(clear_color=(0.10, 0.05, 0.10, 1.0)))
    diff = np.abs(img[..., :3].astype(int) - GOLD["examples/cube"][..., :3].astype(int)).max(axis=2)
    assert np.count_nonzero(diff <= 2) >= 0.99 * diff.size, f"examples/cube: {np.count_nonzero(diff > 2)} px off by > 2 LSB"
    assert diff.mean() < 0.5
    b.close()


def test_oracle_passes_the_goldens_through_the_new_calls():
    check_goldens(load_lights_oracle_backend)


def test_static_light_fields_equal_world_buffer():
    """The sources' light records (view_proj aside) are the bytes world.py's directional_buffer holds."""
    for left in (True, False):
        r = walkthrough_world(left)
        r.set_camera_data(walkthrough_camera(0, left))
        ev = r.evaluate()
        _, lights = ref.evaluate(ev.directional_sources, ev.shadow_target_size[0], ev.shadow_target_size[1], (0.0, 0.0, 0.0), left)
        host = np.frombuffer(ev.directional_buffer[16:], dtype=lights.dtype)
        assert len(host) == len(lights) == 2
        for f in ("color", "direction", "inv_resolution", "atlas_offset", "atlas_size"):
            assert same_words_nan_equal(lights[f], host[f]), f


def check_rejections(b):
    """Every rejected call returns its code and leaves the context as it was."""
    src = ref.sources([((-1.0, -2.0, 0.5), 20.0, 256), ((0.3, -1.0, 0.2), 30.0, 128)])
    b.set_objects(np.zeros(8, dtype=OBJECT_DTYPE))
    with pytest.raises(R3Error) as e:
        b.evaluate_shadow_cameras((0.0, 0.0, 0.0))
    assert e.value.code == R3_E_STATE
    b.set_directional_light_sources(src, ATLAS[0], ATLAS[1], True)
    with pytest.raises(R3Error) as e:
        b.shadow_uniform_upload(0, 8)
    assert e.value.code == R3_E_STATE, "upload before an evaluation"
    b.evaluate_shadow_cameras((1.0, 2.0, 3.0))
    want = b.readback_shadow_cameras(2)
    bad = []
    many = np.zeros(64, dtype=LIGHT_SOURCE_DTYPE)
    many["size"] = 1
    bad.append(many)                                    # more than R3_MAX_SHADOWS
    for field, value in (("size", 0), ("offset", (ATLAS[0] - 63, 0)), ("offset", (0, ATLAS[1] - 63)), ("offset", (2 ** 32 - 1, 0))):
        s = src.copy()
        s[1][field] = value
        bad.append(s)
    for s in bad:
        with pytest.raises(R3Error) as e:
            b.set_directional_light_sources(s, ATLAS[0], ATLAS[1], False)
        assert e.value.code == R3_E_INVALID
    with pytest.raises(R3Error) as e:
        b.set_directional_light_sources(src, 64, 512, False)   # the second map at x = 64 does not fit a 64-wide atlas
    assert e.value.code == R3_E_INVALID
    for idx, count in ((2, 8), (63, 8), (0, 9)):
        with pytest.raises(R3Error) as e:
            b.shadow_uniform_upload(idx, count)
        assert e.value.code == R3_E_INVALID
    with pytest.raises(R3Error) as e:
        b.readback_shadow_cameras(3)
    assert e.value.code == R3_E_INVALID
    got = b.readback_shadow_cameras(2)
    assert same_words_nan_equal(got[0], want[0]) and same_words_nan_equal(got[1], want[1]), "a rejected call changed the cameras or the light buffer"
    b.shadow_uniform_upload(1, 8)
    # r3_set_directional_lights replaces the sources: the device cameras are gone until sources are set again
    b.set_directional_lights(np.zeros(4, np.uint32).tobytes(), ATLAS[0], ATLAS[1])
    for call in (lambda: b.evaluate_shadow_cameras((0.0, 0.0, 0.0)), lambda: b.shadow_uniform_upload(0, 8), lambda: b.readback_shadow_cameras(1)):
        with pytest.raises(R3Error) as e:
            call()
        assert e.value.code == R3_E_STATE


def test_oracle_rejects_invalid_calls_and_keeps_its_state():
    b = load_lights_oracle_backend()
    check_rejections(b)
    b.close()


def test_light_source_layout_matches_c_header():
    import os
    import subprocess
    import tempfile

    fields = LIGHT_SOURCE_DTYPE.names
    prog = "#include <stdio.h>\n#include <stddef.h>\n#include \"r3_layouts.h\"\nint main(void){printf(\"%zu\\n\", sizeof(r3_directional_light_source));"
    prog += "".join(f"printf(\"%zu\\n\", offsetof(r3_directional_light_source, {f}));" for f in fields) + "return 0;}\n"
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "l.c"), os.path.join(d, "l")
        open(src, "w").write(prog)
        subprocess.run(["gcc", "-I", inc, src, "-o", exe], check=True)
        out = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    assert out[0] == LIGHT_SOURCE_DTYPE.itemsize == 48
    assert out[1:] == [LIGHT_SOURCE_DTYPE.fields[f][1] for f in fields]


# ------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_gpu_cameras_equal_oracle_bit_for_bit():
    b = load_cuda_backend(0, parity_target=False)
    check_equals_reference(b)
    b.close()


@pytest.mark.gpu
def test_gpu_rejects_invalid_calls_and_keeps_its_state():
    b = load_cuda_backend(0, parity_target=False)
    check_rejections(b)
    b.close()


@pytest.mark.gpu
def test_gpu_goldens_with_device_cameras():
    check_goldens(lambda: load_cuda_backend(0, parity_target=False))


def frame_products(b, ev, n_lights):
    """Everything the frame leaves that the oracle computes bit for bit, plus the f32 shading result."""
    out = {}
    n = len(ev.object_buffer)
    for cam in [CAMERA_VIEWPORT] + list(range(n_lights)):
        out[f"visible{cam}"] = b.readback_visible(cam).copy()
        out[f"matrices{cam}"] = b.readback_object_matrices(cam, 0, n).copy()
        for part in (0, 1):
            out[f"indices{cam}.{part}"] = b.readback_indices(cam, part).copy()
            out[f"draws{cam}.{part}"] = b.readback_draw_calls(cam, part).copy()
    out["atlas"] = b.readback_shadow_atlas(*ev.shadow_target_size).copy()
    out["depth"] = b.readback_depth().copy()
    return out, b.readback_hdr_f32().copy()


def assert_same_products(a, b, what):
    for k in a:
        assert a[k].shape == b[k].shape and same_words_nan_equal(a[k], b[k]), f"{what}: {k} differs"


def assert_matches_oracle(c, o, what):
    """As test_gpu_parity compares them: the CUDA path sizes its culling buffers by device-side bounds, so the draw records are compared
    over the oracle's count (the rest must be cleared) and the index lists over the ranges those records list."""
    for k in o:
        if k.startswith("draws"):
            assert c[k][:len(o[k])].tobytes() == o[k].tobytes(), f"{what}: {k} differs"
            assert not c[k][len(o[k]):].view(np.uint8).any(), f"{what}: {k} has stray records"
        elif k.startswith("indices"):
            cam, part = k[len("indices"):].split(".")
            if part == "1" and int(cam) != CAMERA_VIEWPORT:
                continue
            for r in o["draws" + k[len("indices"):]]:
                b0, cnt = int(r["base_index"]), int(r["vertex_count"])
                assert np.array_equal(c[k][b0:b0 + cnt], o[k][b0:b0 + cnt]), f"{what}: {k} differs"
        else:
            assert c[k].shape == o[k].shape and same_words_nan_equal(c[k], o[k]), f"{what}: {k} differs"


class CallLog:
    """Wraps a backend and records the entry points a frame calls."""

    def __init__(self, b):
        self.b, self.calls = b, []

    def __getattr__(self, name):
        attr = getattr(self.b, name)
        if callable(attr):
            def wrapped(*a, **k):
                self.calls.append(name)
                return attr(*a, **k)
            return wrapped
        return attr


ENQUEUE_ONLY = {"frame_begin", "frame_end", "clear_shadow_atlas", "set_frame_uniforms", "evaluate_shadow_cameras", "shadow_uniform_upload",
                "object_uniform_upload", "batch_objects", "cull", "shadow_pass", "forward_begin", "forward_pass", "hiz_build", "forward_resolve",
                "forward_blend", "tonemap"}


@pytest.mark.gpu
@pytest.mark.parametrize("left", [True, False])
def test_gpu_walkthrough_with_device_cameras(left):
    """Seven frames of a walkthrough (static world, camera moving across texel boundaries) with two lights, one along -Y, and a
    textured cutout quad in the shadow pass.  Graphed device-camera frames equal eager ones bit for bit and the oracle bit for bit
    (visible lists, MV/MVP, index lists, draw records, atlas, depth) and HDR to 1e-4, never flush after the first frame and call only
    enqueue-only entry points; the host light path fed the numpy R13's light bytes and headers renders the same bits, HDR included."""
    from rend3_b200.routines import BaseRenderGraph

    r = walkthrough_world(left)
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0))
    graph_b, eager_b, host_b = (load_cuda_backend(0, parity_target=True) for _ in range(3))
    orc = load_lights_oracle_backend()
    log = CallLog(graph_b)
    graphs = {id(b): BaseRenderGraph(b) for b in (graph_b, eager_b, host_b, orc)}
    graphs[id(graph_b)] = BaseRenderGraph(log)
    texel = 20.0 / 256
    crossed = set()
    for frame in range(7):
        r.set_camera_data(walkthrough_camera(frame, left))
        ev = r.evaluate()
        up = frame == 0
        flushed = graph_b.frame_graph_stats()["flushed"]
        log.calls = []
        graphs[id(graph_b)].add_to_graph(ev, (256, 144), 1, settings, upload=up, frame_graph=True, device_shadow_cameras=True)
        if frame:
            assert graph_b.frame_graph_stats()["flushed"] == flushed, f"frame {frame} flushed early"
            assert set(log.calls) <= ENQUEUE_ONLY, sorted(set(log.calls) - ENQUEUE_ONLY)
        graphs[id(eager_b)].add_to_graph(ev, (256, 144), 1, settings, upload=up, frame_graph=False, device_shadow_cameras=True)
        graphs[id(orc)].add_to_graph(ev, (256, 144), 1, settings, upload=up, device_shadow_cameras=True)
        # the host path with R13's bytes: r3_set_directional_lights + r3_object_uniform_upload of R13's headers
        loc = ev.camera.location()
        heads, lights = ref.evaluate(ev.directional_sources, ev.shadow_target_size[0], ev.shadow_target_size[1], loc, left)
        dbytes = np.array([len(lights), 0, 0, 0], dtype=np.uint32).tobytes() + lights.tobytes()
        hb, hg = host_b, graphs[id(host_b)]
        if up:
            hg.upload_world(ev)
        hb.set_directional_lights(dbytes, ev.shadow_target_size[0], ev.shadow_target_size[1])

        class HostCameras:
            def __getattr__(self, name):
                return getattr(hb, name)

            def shadow_uniform_upload(self, i, count, mode=3):
                h = heads[i].copy()
                h["object_count"] = count
                hb.object_uniform_upload(i, h, mode)

            def evaluate_shadow_cameras(self, _loc):
                pass

        hg.backend = HostCameras()
        hg.add_to_graph(ev, (256, 144), 1, settings, upload=False, device_shadow_cameras=True)
        hg.backend = hb
        for i, s in enumerate(ev.directional_sources):
            cov = glam.transform_point3(glam.look_at_lh((0, 0, 0), s["direction"], (0, 1, 0)) if left else
                                        glam.look_at_rh((0, 0, 0), s["direction"], (0, 1, 0)), loc)
            crossed.add((i, tuple(np.floor(cov[:2] / texel))))
        pg, hdr_g = frame_products(graph_b, ev, 2)
        pe, hdr_e = frame_products(eager_b, ev, 2)
        po, hdr_o = frame_products(orc, ev, 2)
        ph, hdr_h = frame_products(host_b, ev, 2)
        assert_same_products(pg, pe, f"frame {frame}: graph vs eager")
        assert same_words_nan_equal(hdr_g, hdr_e), f"frame {frame}: graph vs eager HDR"
        assert_matches_oracle(pg, po, f"frame {frame}: device vs oracle")
        assert_same_products(pg, ph, f"frame {frame}: device vs host path")
        assert same_words_nan_equal(hdr_g, hdr_h), f"frame {frame}: device vs host path HDR"
        ok = np.isfinite(hdr_o)
        err = np.abs(hdr_g[ok] - hdr_o[ok]) / np.maximum(1.0, np.abs(hdr_o[ok]))
        assert err.max() <= 1e-4, f"frame {frame}: HDR differs from the oracle by {err.max()}"
        cams, _ = graph_b.readback_shadow_cameras(2)
        assert np.isnan(cams[1]["view_proj"]).any(), "the -Y light's camera is NaN"
        assert len(pg["visible0"]) > 0 and len(pg[f"visible{CAMERA_VIEWPORT}"]) > 0
    assert len({c for c in crossed if c[0] == 0}) >= 3, "the camera crossed texel boundaries of the slanted light"
    stats = graph_b.frame_graph_stats()
    assert stats["frames"] == 7 and stats["graphed"] >= 6 and stats["flushed"] <= 1, stats   # only the first frame may flush (allocations)
    for b in (graph_b, eager_b, host_b, orc):
        b.close()


@pytest.mark.gpu
def test_gpu_switching_light_apis_mid_session():
    """Host lights, then device sources, then host lights again: every frame equals the oracle driven the same way."""
    from rend3_b200.routines import BaseRenderGraph

    r = walkthrough_world(True, cutout=False)
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0))
    b, orc = load_cuda_backend(0, parity_target=True), load_lights_oracle_backend()
    gb, go = BaseRenderGraph(b), BaseRenderGraph(orc)
    for frame, device in enumerate([False, True, True, False, True]):
        r.set_camera_data(walkthrough_camera(frame, True))
        ev = r.evaluate()
        for g in (gb, go):
            g.add_to_graph(ev, (256, 144), 1, settings, upload=True, device_shadow_cameras=device)
        pb, hb = frame_products(b, ev, 2)
        po, ho = frame_products(orc, ev, 2)
        assert_matches_oracle(pb, po, f"frame {frame} (device={device})")
        ok = np.isfinite(ho)
        err = np.abs(hb[ok] - ho[ok]) / np.maximum(1.0, np.abs(ho[ok]))
        assert err.max() <= 1e-4
    b.close()
    orc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("left", [True, False])
def test_gpu_walkthrough_roughness0_grazing_light(left):
    """The walkthrough's quad at roughness 0 (the material default) under the -Y light, which grazes it: n.l is 0 up to rounding,
    and at n.l <= 0 surface_shading is 0 * inf = NaN, which the final max() turns into the ambient term (0 here) for the whole
    pixel.  The kernels normalise the normal with approximations (rsqrtf, contracted products), the oracle exactly, so the two can
    disagree on the sign of n.l.  Everything else is held to the oracle to 1e-4; every pixel that differs more is a quad pixel (its
    alpha is the checker's 230 / 255) where exactly one side fell to the ambient term."""
    from rend3_b200.routines import BaseRenderGraph

    r = walkthrough_world(left, quad_roughness=None)
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0))
    b, orc = load_cuda_backend(0, parity_target=True), load_lights_oracle_backend()
    gb, go = BaseRenderGraph(b), BaseRenderGraph(orc)
    quad_alpha = np.float32(230.0 / 255.0)
    for frame in (0, 3):
        r.set_camera_data(walkthrough_camera(frame, left))
        ev = r.evaluate()
        for g in (gb, go):
            g.add_to_graph(ev, (256, 144), 1, settings, upload=frame == 0, device_shadow_cameras=True)
        pb, hb = frame_products(b, ev, 2)
        po, ho = frame_products(orc, ev, 2)
        assert_matches_oracle(pb, po, f"frame {frame}")
        err = np.abs(hb - ho) / np.maximum(1.0, np.abs(ho))
        bad = (err > 1e-4).any(axis=-1)
        dark_g, dark_o = (hb[..., :3] == 0).all(axis=-1), (ho[..., :3] == 0).all(axis=-1)
        explained = (hb[..., 3] == quad_alpha) & (ho[..., 3] == quad_alpha) & (dark_g != dark_o)
        assert not (bad & ~explained).any(), f"frame {frame}: {int((bad & ~explained).sum())} pixels differ for another reason"
    b.close()
    orc.close()
