"""Cull + bake of transforms whose fourth row is not (0, 0, 0, 1).

The hot copy of a transform keeps rows 0-2 apart from row 3, and the bake substitutes the constant (+0, +0, +0, 1) for row 3
wherever the record's row 3 has exactly those bit patterns.  These cases must take the full path and bake like the oracle word
for word: -0.0 entries, projective rows, NaN, whole non-affine tiles, a lone non-affine slot in an affine tile, and slots that
r3_update_objects moves between affine and non-affine."""
import numpy as np
import pytest

from harness import assert_same_bake
from rend3_b200.backend import CAMERA_VIEWPORT, CB_BAKE, CB_CULL, load_cuda_backend
from rend3_b200.routines import per_camera_header
from rend3_b200.scenes import cloud_camera, object_cloud_records

from oracle import load_oracle_backend

pytestmark = pytest.mark.gpu

ROW3 = [3, 7, 11, 15]          # transform[c * 4 + r]: row 3 of columns 0-3
NEG_ZERO, POS_ZERO = 64, 65     # the same transform with row 3 = (-0, +0, +0, 1) and (+0, +0, +0, 1)


@pytest.fixture()
def cuda():
    b = load_cuda_backend(0)
    yield b
    b.close()


def header_with_negative_row(n):
    """Row 0 of `view` has signs (-, -, -, +): for a column (+0, +0, +0, w) every product of MV row 0 is -0 exactly when w is -0,
    so the sign of w reaches MV."""
    h = per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (1920, 1080), 1, n)
    v = h["view"].reshape(4, 4).copy()          # [column][row]
    v[:, 0] = [-0.5, -0.25, -1.0, 2.0]
    h["view"] = v.reshape(16)
    return h


def non_affine_records(n):
    rec = object_cloud_records(n, seed=31)
    t = rec["transform"]
    rng = np.random.default_rng(32)
    t[0:32, 3:16:4] = rng.uniform(-0.01, 0.01, (32, 4)).astype(np.float32)   # tile 0: every slot projective
    t[0:32, 15] += np.float32(1.0)
    t[40, ROW3] = [0.0, 0.0, 0.0, 2.0]                                       # one non-affine slot inside an affine tile
    t[[NEG_ZERO, POS_ZERO], 0:3] = 0.0                                       # zero xyz in column 0
    t[POS_ZERO] = t[NEG_ZERO]
    t[NEG_ZERO, 3] = np.float32(-0.0)
    t[66, 15] = np.float32(-0.0)                                             # w of column 3 is -0
    t[67, ROW3] = [0.0, np.float32(-0.0), np.float32(-0.0), 1.0]
    t[100, 3] = np.nan
    t[101, 15] = np.nan
    t[n - 1, ROW3] = [0.5, 0.0, 0.0, 1.0]                                    # last slot of a partial tile
    rec["enabled"][[40, 66, 100, 101, n - 1]] = 1
    rec["enabled"][[5, 20]] = [0, 0]                                         # disabled slots in the non-affine tile
    return rec


def test_non_affine_row3_matches_oracle(cuda):
    n = 4096 + 17
    rec = non_affine_records(n)
    header = header_with_negative_row(n)
    orc = load_oracle_backend()
    for b in (cuda, orc):
        b.set_objects(rec)
        b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE | CB_CULL)
    assert_same_bake(cuda, orc, rec, "cull + bake")
    # the -0.0 case can be told apart: the oracle bakes different bits for -0.0 and +0.0 in row 3
    o = orc.readback_object_matrices(CAMERA_VIEWPORT, 0, n).view(np.uint32).reshape(n, 32)
    assert not np.array_equal(o[NEG_ZERO], o[POS_ZERO]), "the chosen view and transform do not separate -0.0 from +0.0"
    for b in (cuda, orc):
        b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE)
    assert_same_bake(cuda, orc, rec, "bake only", culled=False)


def test_update_objects_between_affine_and_non_affine(cuda):
    n = 3000
    rec = non_affine_records(n)
    header = header_with_negative_row(n)
    orc = load_oracle_backend()
    for b in (cuda, orc):
        b.set_objects(rec)
        b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE | CB_CULL)
    assert_same_bake(cuda, orc, rec, "initial")
    slots = np.array([7, 31, 40, 200, 201, 1000, POS_ZERO, n - 1], dtype=np.uint32)
    affine = object_cloud_records(len(slots), seed=33, disabled_fraction=0.0)
    projective = affine.copy()
    projective["transform"][:, ROW3] = [[0.0, 0.0, 0.25, 1.0]] * 4 + [[np.float32(-0.0), 0.0, 0.0, 1.0]] * 4
    steps = [
        ("affine -> non-affine", projective),     # slots 7 / 31 of tile 0 stay non-affine, the others leave the affine path
        ("non-affine -> affine", affine),         # tile 0 gets affine slots, the rest return to the affine path
        ("affine -> non-affine again", projective),
    ]
    for what, new in steps:
        for b in (cuda, orc):
            b.update_objects(slots, new)
            b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE | CB_CULL)
        rec[slots] = new
        assert_same_bake(cuda, orc, rec, what)
