"""Cull + bake of slots whose bounding-sphere centre is not bit for bit the transform's translation.

The cull reads a centred slot's centre from the translation column it already holds for the bake, and only its radius from memory; a
slot whose centre differs in any bit must read the full sphere.  Every planted slot here sits on a frustum plane so that taking the
centre from the translation would flip it: the scenes check this themselves by culling them a second time in the oracle with
sphere_center := translation.  Compared with the oracle word for word: the visible list and every MV / MVP word of enabled slots."""
import numpy as np
import pytest

from harness import assert_same_bake
from rend3_b200.backend import CAMERA_VIEWPORT, CB_BAKE, CB_CULL, load_cuda_backend
from rend3_b200.routines import per_camera_header
from rend3_b200.scenes import cloud_camera, object_cloud_records

from oracle import load_oracle_backend

pytestmark = pytest.mark.gpu

f32 = np.float32
MODE = CB_BAKE | CB_CULL
TRANSLATION = slice(12, 15)          # transform[c * 4 + r]: column 3, rows 0-2


@pytest.fixture()
def cuda():
    b = load_cuda_backend(0)
    yield b
    b.close()


def plane_d(f, p):
    """Plane::distance in the kernel's order, float32 per operation: ((a x + b y) + c z) + d.  f (4,), p (m, 3)."""
    p = np.asarray(p, dtype=f32).reshape(-1, 3)
    return ((f[0] * p[:, 0] + f[1] * p[:, 1]) + f[2] * p[:, 2]) + f[3]


def boundary_spheres(frustum, rng, axis, ulps, count, extent):
    """`count` (translation, centre, radius): the sphere at `centre` touches one frustum plane (distance == -radius) and lies inside the
    others; at `translation` — the centre moved along `axis` by `ulps` ulps (0: by 1e-3 of its magnitude, at least 0.01) — it is outside
    that plane, so a cull that took the centre from the translation would drop it."""
    F = np.asarray(frustum, dtype=f32).reshape(5, 4)
    out = []
    for _ in range(10_000):
        if len(out) == count:
            return out
        k = int(rng.integers(0, 5))
        n = F[k, :3].astype(np.float64)
        if abs(n[axis]) < 0.2 * np.linalg.norm(n):
            continue
        P = rng.uniform(-extent, extent, (4096, 3))
        dP = P @ n + float(F[k, 3])
        C = (P - np.outer(dP / (n @ n), n)).astype(f32)
        dC = plane_d(F[k], C)
        ok = dC < 0                                           # radius -dC > 0
        for j in range(5):
            if j != k:
                ok &= plane_d(F[j], C) >= 1.0
        step = f32(-np.sign(n[axis]))
        for c, d in zip(C[ok], dC[ok]):
            r = f32(-d)
            t = c.copy()
            if ulps:
                for _ in range(ulps):
                    t[axis] = np.nextafter(t[axis], step * f32(np.inf))
            else:
                t[axis] = f32(c[axis] + step * max(f32(0.01), abs(c[axis]) * f32(1e-3)))
            if plane_d(F[k], t)[0] < -r:
                out.append((t, c, r))
                if len(out) == count:
                    break
    raise AssertionError("no sphere on a frustum plane found")


def plant(rec, slots, frustum, rng, axis, ulps=0, extent=1000.0):
    for s, (t, c, r) in zip(np.atleast_1d(slots), boundary_spheres(frustum, rng, axis, ulps, len(np.atleast_1d(slots)), extent)):
        rec["transform"][s, TRANSLATION], rec["sphere_center"][s], rec["sphere_radius"][s], rec["enabled"][s] = t, c, r, 1


def cull(b, rec, camera, header, **kw):
    b.set_objects(rec)
    if "live" in kw:
        n = len(rec)
        b.set_object_sort_info(np.zeros(n, np.uint64), kw["live"], np.zeros((n, 3), f32))
    upload(b, camera, header, len(rec))
    return b.readback_visible(camera)


def upload(b, camera, header, n):
    if camera == CAMERA_VIEWPORT:
        b.object_uniform_upload(CAMERA_VIEWPORT, header, MODE)
    else:
        b.shadow_uniform_upload(camera, n, MODE)


def assert_flips(rec, planted, camera=CAMERA_VIEWPORT, header=None, setup=None, **kw):
    """The scene checks itself: in the oracle, every planted slot's visibility changes when its centre is set to its translation."""
    lists = []
    for centre_from_translation in (False, True):
        r = rec.copy()
        if centre_from_translation:
            r["sphere_center"][planted] = r["transform"][planted, TRANSLATION]
        orc = load_oracle_backend() if setup is None else setup()
        lists.append(cull(orc, r, camera, header, **kw))
        orc.close()
    same = np.isin(planted, lists[0]) == np.isin(planted, lists[1])
    assert not same.any(), f"planted slots {np.asarray(planted)[same][:8]} do not decide their plane"


def centred(rec):
    return np.all(rec["transform"][:, TRANSLATION].view(np.uint32) == rec["sphere_center"].view(np.uint32), axis=1)


def viewport_header(n):
    return per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (1920, 1080), 1, n)


def planted_world(n, frustum, seed=41, extent=1000.0):
    """Records (centred background) with off-centre slots at the placements the kernel treats differently; returns (rec, planted)."""
    rec = object_cloud_records(n, seed=seed)
    rng = np.random.default_rng(seed + 1)
    planted = []
    for s, axis, ulps in ((333, 0, 0), (360, 1, 0), (390, 2, 0), (420, 0, 1), (450, 1, 1), (480, 2, 1)):   # alone in a centred tile
        plant(rec, s, frustum, rng, axis, ulps, extent)
        planted.append(s)
    for i, s in enumerate(range(640, 672)):                                                               # a whole tile
        plant(rec, s, frustum, rng, i % 3, (i // 3) % 2, extent)
        planted.append(s)
    plant(rec, n - 1, frustum, rng, 1, 1, extent)                                                         # last slot of a partial tile
    planted.append(n - 1)
    for s in (900, 1000):                                                                                 # next to disabled slots
        plant(rec, s, frustum, rng, 2, 0, extent)
        planted.append(s)
    rec["enabled"][[899, 901]] = 0
    rec["enabled"][992:1024] = 0
    rec["enabled"][1000] = 1
    # a NaN translation with a finite centre that is inside: a centre taken from the translation would drop it
    plant(rec, 1502, frustum, rng, 0, 0, extent)
    rec["transform"][1502, 12] = np.uint32(0x7fc00123).view(f32)
    planted.append(1502)
    # consistency only (the planted-vs-translation comparison cannot tell these apart): NaN centre equal to the translation's NaN, bit
    # for bit (bit set); NaNs with different payloads (bit clear); -0 against +0 and +0 against -0 (bit clear)
    nan_a, nan_b = np.uint32(0x7fc00001).view(f32), np.uint32(0x7fc00002).view(f32)
    rec["transform"][1500, 12] = nan_a; rec["sphere_center"][1500, 0] = nan_a
    rec["transform"][1501, 12] = nan_a; rec["sphere_center"][1501, 0] = nan_b
    rec["transform"][1503, 12] = f32(-0.0); rec["sphere_center"][1503, 0] = f32(0.0)
    rec["transform"][1504, 13] = f32(0.0); rec["sphere_center"][1504, 1] = f32(-0.0)
    rec["enabled"][1500:1505] = 1
    assert not centred(rec)[np.array(planted + [1501, 1503, 1504])].any() and centred(rec)[1500]
    return rec, np.array(planted)


def test_off_centre_slots_match_oracle(cuda):
    """Every placement, without and with a live mask (r3_set_object_sort_info)."""
    n = 4096 + 21
    header = viewport_header(n)
    rec, planted = planted_world(n, header["frustum"])
    assert_flips(rec, planted, header=header)
    orc = load_oracle_backend()
    for b in (cuda, orc):
        cull(b, rec, CAMERA_VIEWPORT, header)
    assert_same_bake(cuda, orc, rec, "cull + bake")
    live = np.ones(n, np.uint8)
    live[np.random.default_rng(3).random(n) < 0.2] = 0
    live[planted] = 1
    assert_flips(rec, planted, header=header, live=live)
    for b in (cuda, orc):
        cull(b, rec, CAMERA_VIEWPORT, header, live=live)
    assert_same_bake(cuda, orc, rec, "cull + bake with a live mask")
    orc.close()


def test_shadow_camera_off_centre_slots_match_oracle(cuda):
    """The device-camera instantiation (r3_shadow_uniform_upload after r3_evaluate_shadow_cameras)."""
    from oracle.lights import load_lights_oracle_backend
    from shadow_camera_reference import sources

    src = sources([((-1.0, -4.0, 2.0), 40.0, 512)])
    loc = np.array([1.5, 2.0, -3.0], dtype=f32)

    def setup(b=None):
        b = b or load_lights_oracle_backend()
        b.set_directional_light_sources(src, 512, 256, False)
        b.evaluate_shadow_cameras(loc)
        return b

    probe = setup()
    frustum = probe.readback_shadow_cameras(1)[0]["frustum"][0]
    probe.close()
    n = 2048 + 5
    rec, planted = planted_world(n, frustum, seed=43, extent=60.0)
    assert_flips(rec, planted, camera=0, setup=setup)
    orc = setup()
    setup(cuda)
    assert np.array_equal(cuda.readback_shadow_cameras(1)[0]["frustum"], orc.readback_shadow_cameras(1)[0]["frustum"])
    got, want = cull(cuda, rec, 0, None), cull(orc, rec, 0, None)
    assert np.array_equal(got, want), "shadow camera: visible list"
    en = rec["enabled"] != 0
    a = cuda.readback_object_matrices(0, 0, n).view(np.uint32).reshape(n, 32)[en]
    o = orc.readback_object_matrices(0, 0, n).view(np.uint32).reshape(n, 32)[en]
    assert np.array_equal(np.isnan(a.view(f32)), np.isnan(o.view(f32))) and not ((a != o) & ~np.isnan(a.view(f32))).any(), "shadow camera: MV / MVP"
    orc.close()


def test_update_objects_radius_and_moves_between_paths(cuda):
    """r3_update_objects: a centred slot whose radius alone changes (a stale radius array keeps it visible), and slots moved off the
    translation, back onto it and off again over three steps."""
    n = 3000
    header = viewport_header(n)
    F = header["frustum"]
    rng = np.random.default_rng(51)
    rec = object_cloud_records(n, seed=52)
    # slot 77: centred, touching a plane; its radius then shrinks by one ulp, which drops it
    (t, c, r), = boundary_spheres(F, rng, 0, 0, 1, 1000.0)
    rec["transform"][77, TRANSLATION], rec["sphere_center"][77], rec["sphere_radius"][77], rec["enabled"][77] = c, c, r, 1
    orc = load_oracle_backend()
    for b in (cuda, orc):
        cull(b, rec, CAMERA_VIEWPORT, header)
    assert_same_bake(cuda, orc, rec, "initial")
    assert 77 in cuda.readback_visible(CAMERA_VIEWPORT)
    new = rec[[77]].copy()
    new["sphere_radius"] = np.nextafter(new["sphere_radius"], f32(0))
    for b in (cuda, orc):
        b.update_objects(np.array([77], np.uint32), new)
        upload(b, CAMERA_VIEWPORT, header, n)
    rec[77] = new[0]
    assert_same_bake(cuda, orc, rec, "radius only")
    assert 77 not in cuda.readback_visible(CAMERA_VIEWPORT), "the shrunk radius must drop slot 77"

    slots = np.array([5, 31, 32, 600, 601, 602, 1400, n - 1], dtype=np.uint32)
    on_plane = rec[slots].copy()
    plant(on_plane, np.arange(len(slots)), F, rng, 1, 1)
    back = on_plane.copy()
    back["sphere_center"] = back["transform"][:, TRANSLATION]
    for what, new in (("off the translation", on_plane), ("back onto it", back), ("off again", on_plane)):
        trial = rec.copy()
        trial[slots] = new
        if what != "back onto it":
            assert_flips(trial, slots, header=header)
        for b in (cuda, orc):
            b.update_objects(slots, new)
            upload(b, CAMERA_VIEWPORT, header, n)
        rec = trial
        assert_same_bake(cuda, orc, rec, what)
    orc.close()


@pytest.mark.parametrize("form", ["host", "device"])
def test_set_object_transforms_moves_between_paths(cuda, form):
    """r3_set_object_transforms (host and device memory, dense and sparse): mesh spheres centred at the origin give centred world spheres,
    off-centre ones do not; slots cross between the two paths both ways over three steps."""
    import object_transform_case as cases

    from oracle.objtransforms import load_objtransforms_oracle_backend

    n = 4000 + 13
    header = viewport_header(n)
    rec, key, flags, loc, ms = cases.world(n, seed=61, extent=400.0)
    ORIGIN, OFF = np.array([0.0, 0.0, 0.0, 40.0], f32), np.array([5.0, -3.0, 2.0, 0.5], f32)   # a stale radius shows
    at_origin = np.arange(n) < n // 2                         # first half: mesh spheres centred at the mesh origin
    ms = np.where(at_origin[:, None], ORIGIN, OFF).astype(f32)
    orc = load_objtransforms_oracle_backend()
    for b in (cuda, orc):
        b.set_objects(rec)
        b.set_object_sort_info(key, flags, loc)
        b.set_object_mesh_spheres(ms)
    rng = np.random.default_rng(62)
    keep = []
    cur_r, cur_l = rec, loc
    flips = 0
    for step in range(3):
        dense = step == 1
        slots = None if dense else np.sort(rng.choice(n, 1500, replace=False)).astype(np.uint32)
        k = n if dense else len(slots)
        mats = cases.seeded_matrices(k, seed=70 + step, extent=400.0)
        # sparse steps give every moved slot the other kind of mesh sphere: centred slots leave the path and off-centre ones join it
        if not dense:
            at_origin[slots] = ~at_origin[slots]
            ms = np.where(at_origin[:, None], ORIGIN, OFF).astype(f32)
            for b in (cuda, orc):
                b.set_object_mesh_spheres(ms[slots], slots)
        cur_r, cur_l = cases.moved_records(cur_r, cur_l, ms, mats, slots)
        keep.append(cases.apply(cuda, form, mats, slots))
        orc.set_object_transforms(mats, slots)
        for b in (cuda, orc):
            upload(b, CAMERA_VIEWPORT, header, n)
        assert_same_bake(cuda, orc, cur_r, f"step {step} ({'dense' if dense else 'sparse'})")
        c = centred(cur_r)
        assert c.any() and (~c).any()
        r2 = cur_r.copy()
        r2["sphere_center"] = r2["transform"][:, TRANSLATION]
        o2 = load_oracle_backend()
        alt = cull(o2, r2, CAMERA_VIEWPORT, header)
        o2.close()
        flips += int((np.isin(np.arange(n), alt) != np.isin(np.arange(n), cuda.readback_visible(CAMERA_VIEWPORT))).sum())
    assert flips > 0, "no off-centre slot decides its visibility by its centre"
    orc.close()
    del keep


def test_animation_posing_moves_between_paths(cuda):
    """Posed objects (r3_pose_objects refreshes the hot copies through r3_split_slots): every slot starts centred, the posed ones come
    out with off-centre world spheres (the nodes' mesh spheres are off the origin); the cull + bake after the pose equals the oracle's
    on the same records, and some posed slots would flip with their centre taken from the translation."""
    import object_animation_case as anim_cases

    data, jobs, targets, records, loc = anim_cases.case(seed=4, instances=64)
    n = len(records)
    records = records.copy()
    records["sphere_center"] = records["transform"][:, TRANSLATION]
    header = per_camera_header(cloud_camera(pull_back=1.0), CAMERA_VIEWPORT, (640, 360), 1, n)   # side planes cut the crowd
    got_r, _ = anim_cases.run(cuda, data, jobs, targets, records, loc)
    posed = np.zeros(n, bool)
    posed[targets["slot"]] = True
    c = centred(got_r)
    assert c[~posed].all() and (~c[posed]).any()
    orc = load_oracle_backend()
    orc.set_objects(got_r)
    orc.set_object_sort_info(np.zeros(n, np.uint64), np.ones(n, np.uint8), loc)   # run() gave the context sort info: every slot live
    for b in (cuda, orc):
        upload(b, CAMERA_VIEWPORT, header, n)
    assert_same_bake(cuda, orc, got_r, "after the pose")
    orc.close()
    alt = got_r.copy()
    alt["sphere_center"] = alt["transform"][:, TRANSLATION]
    o2 = load_oracle_backend()
    moved = np.isin(np.arange(n), cull(o2, alt, CAMERA_VIEWPORT, header, live=np.ones(n, np.uint8))) != np.isin(np.arange(n), cuda.readback_visible(CAMERA_VIEWPORT))
    o2.close()
    assert moved[posed].any(), "no posed slot decides its visibility by its centre"


def test_resize_growth_then_updates_into_new_slots(cuda):
    """r3_resize_objects with a ragged last word (the new slots' bits start clear), then off-centre and centred records written into
    the new slots."""
    n0, n1 = 1000 + 7, 1000 + 7 + 300
    header = viewport_header(n1)
    F = header["frustum"]
    rng = np.random.default_rng(71)
    rec = object_cloud_records(n1, seed=72)
    orc = load_oracle_backend()
    cuda.set_objects(rec[:n0])
    upload(cuda, CAMERA_VIEWPORT, viewport_header(n0), n0)
    cuda.resize_objects(n1)
    cur = rec.copy()
    cur[n0:] = np.zeros(n1 - n0, dtype=rec.dtype)
    orc.set_objects(cur)                                      # the oracle has no resize: the grown records, zeros past n0
    for b in (cuda, orc):
        upload(b, CAMERA_VIEWPORT, header, n1)
    assert_same_bake(cuda, orc, cur, "grown")
    slots = np.array([n0, n0 + 1, n0 + 24, n0 + 25, n1 - 1], dtype=np.uint32)
    new = rec[slots].copy()
    plant(new, np.arange(3), F, rng, 0, 1)
    new["enabled"] = 1
    trial = cur.copy()
    trial[slots] = new
    assert_flips(trial, slots[:3], header=header)
    for b in (cuda, orc):
        b.update_objects(slots, new)
        upload(b, CAMERA_VIEWPORT, header, n1)
    assert_same_bake(cuda, orc, trial, "updates into the new slots")
    orc.close()
