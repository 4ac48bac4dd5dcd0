"""Skeletons posed by the application — r3_set_joint_matrices and r3_set_joint_matrices_device (Renderer::set_skeleton_joint_matrices /
set_skeleton_joint_transforms) — against the float32 product of tests/anim_reference.py (`_mul`, rule R12) and bit copies, their
validation, their order against r3_pose_skeletons, r3_skin_posed from what they write, and frames through add_to_graph in a frame graph
with the oracle handed the expected joint buffer through r3o_set_skeletons."""
import ctypes
import os

import numpy as np
import pytest

from anim_reference import _mul, same_bits
from harness import ROOT, check_declared_and_exported, expect_error, unbound_backend
from rend3_b200 import glam
from rend3_b200.backend import load_cuda_backend
from rend3_b200.layouts import ATTR_ABSENT, JOINT_WRITE_DTYPE, SKINNING_INPUT_DTYPE

f32 = np.float32
E_INVALID, E_STATE = -1, -5
NO_SKELETONS = np.zeros(0, dtype=SKINNING_INPUT_DTYPE)
# IEEE edges the copy form must keep bit for bit: -0.0, +inf, -inf, quiet NaNs with payloads and sign, a signalling NaN
SPECIAL_BITS = np.array([0x80000000, 0x7F800000, 0xFF800000, 0x7FC01234, 0xFFC00001, 0x7F800001, 0x7FBFFFFF], dtype=np.uint32)


def writes_of(rows):
    """(joint_matrix_base_offset, joint_count, first_matrix, first_inverse_bind) tuples -> JOINT_WRITE_DTYPE records"""
    w = np.zeros(len(rows), dtype=JOINT_WRITE_DTYPE)
    for i, r in enumerate(rows):
        w[i] = r
    return w


def expected(buf, writes, mat4s, inverse_binds=None):
    """The joint buffer after the call: a bit copy of each write's matrices, or glam's global * inverse_bind in float32."""
    out = np.array(buf, dtype=f32).reshape(-1, 16).copy()
    m = np.asarray(mat4s, dtype=f32).reshape(-1, 16)
    with np.errstate(all="ignore"):
        for w in writes:
            base, n, fm, fi = (int(w[f]) for f in JOINT_WRITE_DTYPE.names)
            for k in range(n):
                if inverse_binds is None:
                    out[base + k] = m[fm + k]
                else:
                    ib = np.asarray(inverse_binds, dtype=f32).reshape(-1, 16)[fi + k]
                    out[base + k] = _mul(m[fm + k].reshape(4, 4), ib.reshape(4, 4), f32).reshape(16)
    return out


def random_mats(rng, n, special=True):
    """n affine-ish matrices of mixed magnitude; with `special`, some entries replaced by SPECIAL_BITS"""
    m = rng.uniform(-3, 3, (n, 16)).astype(f32)
    m[:, 3::4] = rng.choice(np.array([0.0, 1.0, 0.5], f32), (n, 4))
    if special and n:
        at = rng.integers(0, m.size, max(1, m.size // 40))
        m.reshape(-1).view(np.uint32)[at] = SPECIAL_BITS[np.arange(len(at)) % len(SPECIAL_BITS)]
    return m


# (joint_count, first_matrix) per write; the two writes of 33 read one source range, as rend3's armature primitives do
COUNTS = [0, 1, 31, 32, 33, 33, 65, 600]


def copy_case(seed=0):
    """A joint buffer with a gap before and after every destination, the writes of COUNTS, and their sources."""
    rng = np.random.default_rng(seed)
    rows, base, src = [], 3, 0
    for i, n in enumerate(COUNTS):
        first = rows[-1][2] if i == 5 else src   # the second 33-joint write shares the first one's source range
        rows.append((base, n, first, first))
        base += n + 2
        if i != 5:
            src += n
    buf = random_mats(rng, base + 3, special=False)
    return buf, writes_of(rows), random_mats(rng, src + 5), random_mats(rng, src + 5, special=False)


# ------------------------------------------------------------------ without a GPU
def test_library_exports_both_entry_points_with_the_headers_signatures():
    check_declared_and_exported(("int r3_set_joint_matrices(r3_ctx*, const r3_joint_write* writes, uint32_t n_writes, const float* mat4s, "
                                 "uint32_t n_mat4s, const float* inverse_binds_or_null, uint32_t n_inverse_binds);",
                                 "int r3_set_joint_matrices_device(r3_ctx*, const r3_joint_write* d_writes, uint32_t n_writes, const float* d_mat4s, "
                                 "uint32_t n_mat4s, const float* d_inverse_binds_or_null, uint32_t n_inverse_binds);"),
                                (None, None, 0, None, 0, None, 0))


def test_joint_write_layout_matches_c_header():
    import subprocess
    import tempfile

    src = "\n".join(["#include <stdio.h>", "#include <stddef.h>", f'#include "{ROOT}/include/r3_layouts.h"', "int main(void){",
                     'printf("size %zu\\n", sizeof(r3_joint_write));']
                    + [f'printf("{f} %zu\\n", offsetof(r3_joint_write, {f}));' for f in JOINT_WRITE_DTYPE.names] + ["return 0;}"])
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(c, "w").write(src)
        subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", c, "-o", exe], check=True)
        out = dict(l.split() for l in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out["size"]) == JOINT_WRITE_DTYPE.itemsize == 16
    assert [int(out[f]) for f in JOINT_WRITE_DTYPE.names] == [0, 4, 8, 12]
    assert 'R3_STATIC_ASSERT(sizeof(r3_joint_write) == 16, "r3_joint_write");' in open(os.path.join(ROOT, "include", "r3_layouts.h")).read()


W1 = writes_of([(0, 1, 0, 0)])


@pytest.mark.parametrize("writes,mat4s,inverse_binds", [
    (np.zeros(4, np.uint32), np.zeros((1, 16), f32), None),            # words, not records
    (np.zeros((1, 1), JOINT_WRITE_DTYPE), np.zeros((1, 16), f32), None),  # 2-d records
    (W1, np.zeros((1, 16), np.float64), None),                         # float64 matrices
    (W1, np.zeros(16, f32), None),                                     # 1-d matrices
    (W1, np.zeros((1, 12), f32), None),                                # 12 floats per matrix
    (W1, np.zeros((1, 16), f32), np.zeros((1, 3, 4), f32)),            # 3 x 4 inverse binds
    (W1, np.zeros((1, 16), f32), np.zeros((1, 16), np.int32)),         # integer inverse binds
], ids=["words", "2d-writes", "float64", "1d-mats", "12-floats", "3x4-binds", "int-binds"])
def test_host_wrapper_rejects_bad_shapes_and_dtypes_before_calling(writes, mat4s, inverse_binds):
    with pytest.raises(AssertionError, match="writes|mat4s|inverse_binds"):
        unbound_backend().set_joint_matrices(writes, mat4s, inverse_binds)


class _FakeCuda:
    """Just enough of a CUDA tensor for the wrapper's checks (no device needed)."""

    def __init__(self, shape, dtype, ptr=4096, contiguous=True, cuda=True):
        self.shape, self.dtype, self._ptr, self._contiguous, self.is_cuda = tuple(shape), dtype, ptr, contiguous, cuda

    def dim(self):
        return len(self.shape)

    def numel(self):
        return int(np.prod(self.shape))

    def element_size(self):
        return {"torch.float32": 4, "torch.int32": 4, "torch.uint8": 1, "torch.float64": 8}[self.dtype]

    def is_floating_point(self):
        return self.dtype.startswith("torch.float")

    def is_contiguous(self):
        return self._contiguous

    def data_ptr(self):
        return self._ptr


def test_device_wrapper_rejects_host_misaligned_and_mistyped_tensors_before_calling():
    b = unbound_backend()
    w, m = _FakeCuda((2, 4), "torch.int32"), _FakeCuda((2, 16), "torch.float32")
    bad = [
        (_FakeCuda((2, 4), "torch.int32", cuda=False), m, None),                   # host writes
        (w, _FakeCuda((2, 16), "torch.float32", cuda=False), None),                # host matrices
        (w, _FakeCuda((2, 16), "torch.float32", ptr=4100), None),                  # matrices 4-byte aligned only
        (w, m, _FakeCuda((2, 16), "torch.float32", ptr=4104)),                     # inverse binds 8-byte aligned only
        (w, _FakeCuda((2, 16), "torch.float32", contiguous=False), None),          # strided matrices
        (w, _FakeCuda((2, 16), "torch.float64"), None),                            # float64 matrices
        (w, _FakeCuda((2, 12), "torch.float32"), None),                            # 12 floats per matrix
        (_FakeCuda((2, 4), "torch.float32"), m, None),                             # float writes
        (_FakeCuda((2, 3), "torch.int32"), m, None),                               # 12-byte writes
        (np.zeros(2, JOINT_WRITE_DTYPE), m, None),                                 # a numpy array
        (4096, m, None),                                                           # a raw pointer without its count
    ]
    for writes, mat4s, ib in bad:
        with pytest.raises(AssertionError):
            b.set_joint_matrices_device(writes, mat4s, ib)


# ------------------------------------------------------------------ GPU
def upload(b, buf, inputs=NO_SKELETONS):
    b.set_skeletons(inputs, buf)
    return b


def bits(a):
    return np.ascontiguousarray(a, dtype=f32).view(np.uint32)


@pytest.mark.gpu
def test_gpu_copy_form_keeps_every_bit():
    buf, writes, mats, _ = copy_case(1)
    b = upload(load_cuda_backend(0), buf)
    b.set_joint_matrices(writes, mats)
    got = b.readback_joint_matrices(0, len(buf))
    b.close()
    want = expected(buf, writes, mats)
    assert np.array_equal(bits(got), bits(want)), f"{np.count_nonzero(bits(got) != bits(want))} words differ"
    assert np.isin(bits(got), SPECIAL_BITS).sum() >= len(SPECIAL_BITS), "the IEEE edges reached the buffer"
    written = np.zeros(len(buf), bool)
    for w in writes:
        written[int(w["joint_matrix_base_offset"]): int(w["joint_matrix_base_offset"]) + int(w["joint_count"])] = True
    assert np.array_equal(bits(got)[~written], bits(buf)[~written]), "ranges no write names keep r3_set_skeletons' matrices"


@pytest.mark.gpu
def test_gpu_product_form_equals_float32_restatement():
    buf, writes, mats, binds = copy_case(2)
    writes["first_inverse_bind"][-1] = writes["first_inverse_bind"][-2] = 0   # the 65- and 600-joint writes share one inverse-bind range
    b = upload(load_cuda_backend(0), buf)
    b.set_joint_matrices(writes, mats, binds)
    got = b.readback_joint_matrices(0, len(buf))
    b.close()
    want = expected(buf, writes, mats, binds)
    assert same_bits(got, want), f"{np.count_nonzero(bits(got) != bits(want))} words differ"
    assert np.isnan(want).any() and np.isfinite(want).mean() > 0.5


def _device_sources(b, *arrays):
    """Each array as a CUDA tensor produced by a torch op on the context's stream."""
    import torch

    stream = torch.cuda.ExternalStream(b.stream())
    staged = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        out = [s.clone() for s in staged]
    stream.synchronize()   # other contexts' streams read them too
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("product", [False, True], ids=["copy", "product"])
def test_gpu_device_form_equals_host_form_and_drops_bad_writes_whole(product):
    buf, writes, mats, binds = copy_case(3)
    n_buf, n_m = len(buf), len(mats)
    bad = writes_of([(n_buf - 2, 3, 0, 0),                 # destination runs past the joint buffer
                     (0xFFFFFFFF, 2, 0, 0),                # destination whose 32-bit end wraps
                     (0, 4, n_m - 3, 0),                   # source past the matrices
                     (0, 2, 0xFFFFFFFF, 0)]                # source whose 32-bit end wraps
                    + ([(0, 4, 0, n_m - 2), (0, 2, 0, 0xFFFFFFFF)] if product else []))
    mixed = np.concatenate([bad[:2], writes[:4], bad[2:], writes[4:]])
    ib = binds if product else None
    host = upload(load_cuda_backend(0), buf)
    host.set_joint_matrices(writes, mats, ib)
    want = host.readback_joint_matrices(0, n_buf)
    host.close()
    dev = upload(load_cuda_backend(0), buf)
    d = _device_sources(dev, mixed.view(np.int32).reshape(-1, 4), mats, binds)
    dev.set_joint_matrices_device(d[0], d[1], d[2] if product else None)
    got = dev.readback_joint_matrices(0, n_buf)
    # misaligned matrices are refused before anything is enqueued
    expect_error(E_INVALID, dev.set_joint_matrices_device, d[0].data_ptr(), d[1].data_ptr() + 4, None, n_writes=len(mixed), n_mat4s=2)
    expect_error(E_INVALID, dev.set_joint_matrices_device, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr() + 8, n_writes=len(mixed),
                 n_mat4s=2, n_inverse_binds=2)
    assert np.array_equal(bits(dev.readback_joint_matrices(0, n_buf)), bits(got))
    dev.close()
    assert np.array_equal(bits(got), bits(want)), f"{np.count_nonzero(bits(got) != bits(want))} words differ"
    assert same_bits(got, expected(buf, writes, mats, ib))


@pytest.mark.gpu
def test_gpu_rejections_leave_the_buffer_unchanged():
    buf, writes, mats, binds = copy_case(4)
    b = load_cuda_backend(0)
    expect_error(E_STATE, b.set_joint_matrices, writes, mats)
    expect_error(E_STATE, b.set_joint_matrices_device, 4096, 4096, None, n_writes=1, n_mat4s=1)
    upload(b, buf)
    n_buf, n_m = len(buf), len(mats)
    cases = {
        "destination past the buffer": (writes_of([(0, 2, 0, 0), (n_buf - 1, 2, 0, 0)]), binds),
        "destination end wraps in 32 bits": (writes_of([(0xFFFFFFFF, 2, 0, 0)]), None),
        "source past the matrices": (writes_of([(0, 4, n_m - 3, 0)]), None),
        "source end wraps in 32 bits": (writes_of([(0, 2, 0xFFFFFFFF, 0)]), None),
        "source past the inverse binds": (writes_of([(0, 4, 0, len(binds) - 3)]), binds),
        "overlapping destinations": (writes_of([(10, 5, 0, 0), (0, 3, 0, 0), (14, 2, 0, 0)]), None),
        "one destination named twice": (writes_of([(7, 1, 0, 0), (7, 1, 1, 0)]), None),
    }
    for what, (w, ib) in cases.items():
        expect_error(E_INVALID, b.set_joint_matrices, w, mats, ib)
        assert np.array_equal(bits(b.readback_joint_matrices(0, n_buf)), bits(buf)), what
    fn, m, w = b._fn("set_joint_matrices"), np.ascontiguousarray(mats), np.ascontiguousarray(writes)
    u = ctypes.c_uint32
    for what, args in {"null writes": (None, u(1), m.ctypes.data, u(len(m)), None, u(0)),
                       "null matrices": (w.ctypes.data, u(len(w)), None, u(len(m)), None, u(0)),
                       "null inverse binds with a count": (w.ctypes.data, u(len(w)), m.ctypes.data, u(len(m)), None, u(3))}.items():
        assert fn(b.ctx, *(ctypes.c_void_p(a) if isinstance(a, int) else a for a in args)) == E_INVALID, what
        assert np.array_equal(bits(b.readback_joint_matrices(0, n_buf)), bits(buf)), what
    # a zero-count write may sit anywhere and overlap anything
    b.set_joint_matrices(writes_of([(n_buf, 0, 0, 0), (3, 0, 0, 0), (0xFFFFFFFF, 0, 0xFFFFFFFF, 0)]), mats)
    b.set_joint_matrices(writes_of([]), mats)
    assert np.array_equal(bits(b.readback_joint_matrices(0, n_buf)), bits(buf))
    b.close()


@pytest.mark.gpu
def test_gpu_later_of_pose_and_write_wins():
    import animation_case as cases

    library, jobs, targets, buf = cases.case("humanoid", 65, seed=4)
    t0, n0 = int(targets["joint_matrix_base_offset"][0]), int(targets["joint_count"][0])
    assert n0 >= 20
    targeted = np.zeros(len(buf), bool)
    for tg in targets:
        targeted[int(tg["joint_matrix_base_offset"]): int(tg["joint_matrix_base_offset"]) + int(tg["joint_count"])] = True
    free = int(np.flatnonzero(~targeted)[0])
    rng = np.random.default_rng(6)
    mats = random_mats(rng, 12, special=False)
    writes = writes_of([(t0 + 5, 10, 0, 0), (free, 1, 11, 0)])   # inside target 0's range, and a range no job targets

    def run(order):
        b = load_cuda_backend(0)
        b.set_animations(*library.arrays())
        b.set_skeletons(NO_SKELETONS, buf)
        b.set_pose_jobs(jobs, targets)
        for step in order:
            b.pose_skeletons() if step == "pose" else b.set_joint_matrices(writes, mats)
        out = b.readback_joint_matrices(0, len(buf))
        b.close()
        return out

    posed = run(["pose"])
    both = expected(posed, writes, mats)
    assert same_bits(run(["pose", "write"]), both), "pose then write: the write wins on its range"
    after = run(["write", "pose"])
    want = posed.copy()
    want[free] = mats[11]
    assert same_bits(after, want), "write then pose: the pose wins where a job writes, the write stays elsewhere"
    assert not same_bits(posed[t0 + 5:t0 + 15], mats[:10])


def _two_skeletons(seed):
    import skinning_case

    words, inputs, _, _ = skinning_case.build(seed=seed, vertex_counts=(257, 3000), joints_per_skeleton=(30, 30))
    inputs["joint_matrix_base_offset"] = [2, 40]   # buffer of 72 matrices: gaps before, between and after
    return words, inputs


@pytest.mark.gpu
def test_gpu_skin_posed_from_written_matrices_equals_skin_and_oracle():
    """r3_skin_posed after the writes == r3_skin(records, the same matrices) == the oracle's skinning of that buffer."""
    from oracle.anim import load_anim_oracle_backend

    words, inputs = _two_skeletons(8)
    rng = np.random.default_rng(8)
    globals_ = np.array([glam.from_scale_rotation_translation(rng.uniform(0.5, 2, 3), q / np.linalg.norm(q), rng.uniform(-2, 2, 3))
                         for q in rng.standard_normal((30, 4))], dtype=f32).reshape(-1, 16)
    binds = np.array([glam.from_scale_rotation_translation(rng.uniform(0.5, 2, 3), q / np.linalg.norm(q), rng.uniform(-2, 2, 3))
                      for q in rng.standard_normal((30, 4))], dtype=f32).reshape(-1, 16)
    writes = writes_of([(2, 30, 0, 0), (40, 30, 0, 0)])   # both skeletons from one source range (the armature case)
    start = np.zeros((72, 16), f32)
    want = expected(start, writes, globals_, binds)
    assert np.isfinite(want).all()
    b = upload(load_cuda_backend(0), start, inputs)
    b.set_mesh_buffer(words)
    b.set_joint_matrices(writes, globals_, binds)
    b.skin_posed()
    mesh, jm = b.readback_mesh_buffer(len(words)), b.readback_joint_matrices(0, 72)
    b.close()
    assert np.array_equal(bits(jm), bits(want))
    ref = load_cuda_backend(0)
    ref.set_mesh_buffer(words)
    ref.skin(inputs, want)
    assert np.array_equal(ref.readback_mesh_buffer(len(words)), mesh)
    ref.close()
    orc = load_anim_oracle_backend()
    orc.set_mesh_buffer(words)
    orc.set_skeletons(inputs, want)
    orc.skin_posed()
    assert np.array_equal(orc.readback_mesh_buffer(len(words)), mesh)
    orc.close()
    assert not np.array_equal(mesh, words)


# ---- frames: the reference skinning example's motion on a two-bone cylinder
BIND_0 = glam.from_translation((0.0, 0.0, -4.18))
INVERSE_BINDS = np.array([glam.from_translation((0.0, 0.0, 4.18)), glam.identity()], dtype=f32).reshape(2, 16)


def example_globals(t):
    """examples/src/skinning/mod.rs:38-54: joint 0 at from_translation(0, 0, -4.18), joint 1 at from_translation(0) *
    from_rotation_x(30 sin(5 t) degrees)."""
    angle = np.radians(f32(30.0) * f32(np.sin(f32(5.0) * f32(t))))
    return np.array([BIND_0, glam.mul(glam.from_translation((0.0, 0.0, 0.0)), glam.from_rotation_x(angle))], dtype=f32).reshape(2, 16)


def cylinder_world(resolution):
    """One cylinder of radius 0.5 along z in [-4, 4] (bone 0 below z = 0, bone 1 above, blended across z in [-0.5, 0.5]), a directional
    light with a shadow map, a camera to its side.  Returns (EvalOutput, its one r3_skinning_input): the position range of the mesh is
    skinned in place from a copy appended to the mesh buffer."""
    from rend3_b200.scenes import bulk_object_records, eval_with_bulk_objects
    from rend3_b200.world import LEFT, Camera, DirectionalLight, MeshBuilder, PbrMaterial, Renderer

    rings, seg = 17, 16
    z = np.linspace(-4.0, 4.0, rings).astype(f32)
    a = np.linspace(0, 2 * np.pi, seg, endpoint=False)
    pos = np.array([(0.5 * np.cos(t), 0.5 * np.sin(t), zz) for zz in z for t in a], dtype=f32)
    idx = []
    for r in range(rings - 1):
        for s in range(seg):
            p, q = r * seg + s, r * seg + (s + 1) % seg
            idx += [p, q, p + seg, q, q + seg, p + seg]
    r = Renderer(LEFT, aspect_ratio=resolution[0] / resolution[1])
    mesh = r.add_mesh(MeshBuilder.new(pos, LEFT).with_indices(np.array(idx, np.uint32)).build())
    r.add_material(PbrMaterial(albedo_value=(0.8, 0.5, 0.3, 1.0), roughness_factor=0.5))
    r.set_camera_data(Camera(("perspective", 60.0, 0.1), glam.look_at_lh((11.0, 2.0, 0.5), (0.0, 0.0, 0.0), (0.0, 1.0, 0.0))))
    r.add_directional_light(DirectionalLight(color=(1, 1, 1), intensity=1.0, direction=(-1.0, -4.0, 2.0), distance=30.0, resolution=512))
    mesh_ids = np.array([mesh, mesh], np.int64)
    transforms = np.array([glam.identity(), glam.from_translation((0.0, -2.5, 3.0))], dtype=f32)
    rec, loc = bulk_object_records(r, transforms, mesh_ids, np.zeros(2, np.uint32))
    ev = eval_with_bulk_objects(r, rec, loc, 2, mesh_ids)
    pos_off = int(ev.object_buffer["attr_offset"][0][0])
    nv = len(pos)
    w1 = np.clip((pos[:, 2] + 0.5) / 1.0, 0.0, 1.0).astype(f32)
    weights = np.stack([1 - w1, w1, np.zeros(nv, f32), np.zeros(nv, f32)], axis=1).astype(f32)
    joints = np.tile(np.array([0, 1, 0, 0], np.uint16), (nv, 1))
    base = len(ev.mesh_buffer)
    ev.mesh_buffer = np.concatenate([ev.mesh_buffer, pos.view(np.uint32).reshape(-1), joints.view(np.uint32).reshape(-1),
                                     weights.view(np.uint32).reshape(-1)])
    skel = np.zeros(1, dtype=SKINNING_INPUT_DTYPE)
    skel["base_position_offset"] = 4 * base
    skel["joint_indices_offset"] = 4 * (base + 3 * nv)
    skel["joint_weight_offset"] = 4 * (base + 5 * nv)
    skel["updated_position_offset"] = pos_off
    for f in ("base_normal_offset", "base_tangent_offset", "updated_normal_offset", "updated_tangent_offset"):
        skel[f] = ATTR_ABSENT
    skel["vertex_count"] = nv
    skel["joint_matrix_base_offset"] = 0
    return ev, skel


def cylinder_clip():
    """A clip over the cylinder's two joints for the posed variant: joint 1 swings about x, joint 0 holds its bind translation."""
    from rend3_b200.animation import Animation, AnimationData, Node, NodeChannels, Skin, Track

    nodes = [Node(None, (0.0, 0.0, -4.18)), Node(None)]
    q = [np.array([np.sin(h), 0, 0, np.cos(h)], f32) for h in (0.0, 0.3, -0.2)]
    hold = np.array([[0.0, 0.0, -4.18]] * 2, f32)   # an unanimated joint would be IDENTITY, not its bind pose (lib.rs:219)
    tracks = {0: NodeChannels(translation=Track(np.array([0, 2], f32), hold)),
              1: NodeChannels(rotation=Track(np.array([0, 1, 2], f32), np.array(q, f32)))}
    return AnimationData(nodes, [Skin([0, 1], INVERSE_BINDS.copy())], [Animation(tracks, 2.0)])


@pytest.mark.gpu
@pytest.mark.parametrize("samples,posed", [(1, False), (4, False), (1, True)], ids=["1x", "4x", "1x-posed-override"])
def test_gpu_frames_with_device_joint_matrices_stay_one_graph(samples, posed):
    """Six frames through add_to_graph(joint_matrices=<CUDA tensors>, frame_graph=True), the matrices changing every frame: no early
    flush, the same bits as the same frames run eagerly, the expected joint buffer, the oracle's skinned mesh word for word and its
    shading within 1e-4.  The joint buffer also holds a second skeleton's range written from the same sources (rend3's armature).  With
    `posed`, a clip poses both joints first and the write overrides joint 1 (a ragdoll over the clip)."""
    import torch
    from oracle.anim import load_anim_oracle_backend
    from rend3_b200.backend import load_cuda_backend
    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings

    res = (256, 144)
    ev, skel = cylinder_world(res)
    data = cylinder_clip() if posed else None
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0))
    graph_b, eager_b, orc = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True), load_anim_oracle_backend()
    runs = [(graph_b, True), (eager_b, False), (orc, False)]
    graphs = {id(b): BaseRenderGraph(b) for b, _ in runs}
    # the joint buffer: the cylinder's skeleton at 0, a second skeleton's range at 2 reading the same sources
    writes = writes_of([(1, 1, 1, 1), (3, 1, 1, 1)] if posed else [(0, 2, 0, 0), (2, 2, 0, 0)])

    def oracle_set_joint_matrices(w, m, ib):
        """the oracle has no such call: it gets the restated buffer through r3o_set_skeletons (which also drops its pose jobs)"""
        orc.set_skeletons(skel, expected(orc.readback_joint_matrices(0, 4), w, m, ib))
    orc.set_joint_matrices = oracle_set_joint_matrices

    def jobs(t):
        return data.pose_jobs([(0, t, {0: [(0, 2), (2, 2)]})])

    for b, _ in runs:   # a first, eager frame allocates the render targets and culling buffers
        graphs[id(b)].upload_world(ev)
        b.set_skeletons(skel, np.zeros((4, 16), f32))
        if posed:
            b.set_animations(*data.library.arrays())
            b.set_pose_jobs(*jobs(0.0))
        graphs[id(b)].add_to_graph(ev, res, samples, settings, upload=False, posed_skinning=posed,
                                   joint_matrices=(writes, example_globals(0.0), INVERSE_BINDS), frame_graph=False)
    ref_buf = orc.readback_joint_matrices(0, 4)
    keep = []
    for frame, t in enumerate([0.05, 0.2, 0.33, 0.5, 0.71, 0.9]):
        mats = example_globals(t)
        d_writes, d_mats, d_binds = _device_sources(graph_b, writes.view(np.int32).reshape(-1, 4), mats, INVERSE_BINDS)
        keep.append((d_writes, d_mats, d_binds))
        flushed = graph_b.frame_graph_stats()["flushed"]
        out = []
        for b, fg in runs:
            if posed:
                b.set_pose_jobs(*jobs(t))
            jm = (d_writes, d_mats, d_binds) if b is not orc else (writes, mats, INVERSE_BINDS)
            graphs[id(b)].add_to_graph(ev, res, samples, settings, upload=False, posed_skinning=posed, joint_matrices=jm, frame_graph=fg)
            out.append((b.readback_hdr_f32().copy(), b.readback_mesh_buffer(len(ev.mesh_buffer)), b.readback_joint_matrices(0, 4)))
        assert graph_b.frame_graph_stats()["flushed"] == flushed, f"frame {frame} flushed early"
        (hg, mg, jg), (he, me, je), (ho, mo, jo) = out
        assert np.array_equal(hg.view(np.uint32), he.view(np.uint32)) and np.array_equal(mg, me) and np.array_equal(bits(jg), bits(je)), \
            f"frame {frame}: graph != eager"
        if not posed:
            assert np.array_equal(bits(jg), bits(expected(ref_buf, writes, mats, INVERSE_BINDS))), f"frame {frame}: joint buffer"
        assert np.array_equal(bits(jg[[1, 3]]), bits(expected(np.zeros((4, 16), f32), writes, mats, INVERSE_BINDS)[[1, 3]])), \
            f"frame {frame}: joint 1 is the application's"
        assert same_bits(jg, jo) and np.array_equal(mg, mo), f"frame {frame}: joint buffer / skinned mesh differ from the oracle"
        err = np.abs(hg - ho) / np.maximum(1.0, np.abs(ho))
        assert err.max() <= 1e-4, f"frame {frame}: shading differs from the oracle by {err.max()}"
    stats = graph_b.frame_graph_stats()
    assert stats["graphed"] == 6 and stats["flushed"] == 0, stats
    assert not np.array_equal(out[0][1], ev.mesh_buffer), "the cylinder was skinned"
    for b, _ in runs:
        b.close()
    torch.cuda.synchronize()
