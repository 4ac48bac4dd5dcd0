"""ctypes binding of the C ABI declared in include/rend3_b200.h.

`Backend` wraps one context of a shared library exporting that ABI.  The product library is
librend3_b200.so (prefix ``r3_``); loading it is `load_cuda_backend()`.  The test suite binds
its CPU checker through the same class with another prefix — this module knows nothing about
it and never falls back to it: if the CUDA library is missing, loading fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

from .layouts import (
    BATCH_DTYPE,
    CAMERA_HEADER_DTYPE,
    INDIRECT_CALL_DTYPE,
    OBJECT_MATRICES_DTYPE,
    REGION_DTYPE,
)

CAMERA_VIEWPORT = 0xFFFFFFFF
CB_BAKE, CB_CULL = 1, 2

_ROOT = os.path.dirname(os.path.abspath(__file__))
CUDA_LIB_PATH = os.path.join(_ROOT, "librend3_b200.so")

# every entry point of include/rend3_b200.h (tests check the .so exports all of them)
ENTRY_POINTS = [
    "abi_version", "ctx_create", "ctx_destroy", "last_error", "sync", "get_stream", "launch_count", "set_stage_timing", "stage_times", "frame_begin", "frame_end", "frame_graph_stats",
    "set_objects", "update_objects", "set_objects_device", "set_object_sort_info", "set_mesh_buffer", "set_textures", "set_skybox",
    "set_materials", "set_directional_lights", "set_point_lights", "set_frame_uniforms",
    "object_uniform_upload", "visible_count", "readback_visible", "readback_object_matrices",
    "batch_objects", "batch_counts", "readback_batches", "batching_info", "cull", "readback_indices",
    "readback_draw_calls", "readback_culling_results", "set_render_target", "clear_shadow_atlas",
    "shadow_pass", "forward_begin", "forward_pass", "hiz_build", "forward_resolve", "forward_blend", "tonemap",
    "set_parity_target", "readback_hdr_f32", "readback_hdr_f16", "readback_depth", "readback_ldr", "readback_shadow_atlas",
    "readback_hiz", "forward_stats", "forward_light_evaluations", "device_ptr", "set_scissor_rows", "skin", "readback_mesh_buffer",
    "exchange_create", "exchange_connect", "exchange_words", "exchange_merge", "exchange_merged", "exchange_count", "exchange_counts", "exchange_destroy",
    "peer_create", "peer_connect", "peer_send_atlas_rect", "peer_send_rows", "peer_signal", "peer_wait", "peer_destroy", "clear_shadow_rect", "set_cull_shard",
    "update_object_sort_info", "resize_objects", "update_mesh_buffer", "update_textures",
    "set_animations", "set_skeletons", "set_pose_jobs", "pose_skeletons", "skin_posed", "readback_joint_matrices",
    "set_object_animations", "set_object_pose_jobs", "pose_objects", "readback_objects",
    "set_object_mesh_spheres", "set_object_transforms", "set_object_transforms_device",
    "set_objects_enabled", "set_objects_enabled_device",
    "update_materials", "update_materials_device", "readback_materials",
    "set_joint_matrices", "set_joint_matrices_device",
    "set_deformable_meshes", "deform_meshes", "deform_meshes_device", "readback_deformable_mesh_spheres",
    "set_remeshable_meshes", "remesh_meshes", "remesh_meshes_device", "readback_remesh_status", "debug_invocation_bound",
    "set_object_variants", "switch_object_variants", "switch_object_variants_device", "readback_object_variants",
    "update_directional_light_sources", "update_directional_light_sources_device",
    "write_texture_regions", "write_texture_regions_device", "readback_texels",
]


class _AnimLibrary(C.Structure):
    """r3_anim_library (include/rend3_b200.h)"""
    _fields_ = [("skins", C.c_void_p), ("n_skins", C.c_uint32), ("joints", C.c_void_p), ("n_joints", C.c_uint32), ("order", C.c_void_p),
                ("clips", C.c_void_p), ("n_clips", C.c_uint32), ("channels", C.c_void_p), ("n_channels", C.c_uint32),
                ("keys", C.c_void_p), ("n_keys", C.c_uint64)]


class _AnimObjectLibrary(C.Structure):
    """r3_anim_object_library (include/rend3_b200.h)"""
    _fields_ = [("nodes", C.c_void_p), ("n_nodes", C.c_uint32), ("clips", C.c_void_p), ("n_clips", C.c_uint32), ("channels", C.c_void_p),
                ("n_channels", C.c_uint32), ("keys", C.c_void_p), ("n_keys", C.c_uint64), ("left_handed", C.c_uint32)]


class R3Error(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"rend3_b200 error {code}: {message}")
        self.code = code


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _u32_list(a, what: str) -> np.ndarray:
    """A 1-d integer array inside the uint32 range, as contiguous uint32."""
    a = np.asarray(a)
    assert a.ndim == 1 and a.dtype.kind in "iu", f"{what}: a 1-d integer array"
    assert not len(a) or (a.min() >= 0 and a.max() <= 0xFFFFFFFF), f"{what}: out of the uint32 range"
    return np.ascontiguousarray(a, dtype=np.uint32)


class Backend:
    """One context.  Method names follow the C ABI one to one."""

    def __init__(self, lib: C.CDLL, prefix: str = "r3_", device: int = 0):
        self.lib, self.prefix = lib, prefix
        self.ctx = C.c_void_p()
        self._fn("last_error").restype = C.c_char_p
        self._fn("abi_version").restype = C.c_uint32
        rc = self._fn("ctx_create")(C.c_int(device), C.byref(self.ctx))
        if rc != 0:
            raise R3Error(rc, "context creation failed (no CUDA device?)")

    def _fn(self, name):
        return getattr(self.lib, self.prefix + name)

    def _call(self, name, *args):
        rc = self._fn(name)(self.ctx, *args)
        if rc != 0:
            raise R3Error(rc, (self._fn("last_error")(self.ctx) or b"?").decode())

    def close(self):
        if self.ctx:
            self._fn("ctx_destroy")(self.ctx)
            self.ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- context
    def sync(self):
        self._call("sync")

    def stream(self) -> int:
        s = C.c_void_p()
        self._call("get_stream", C.byref(s))
        return s.value or 0

    def launch_count(self) -> int:
        n = C.c_uint64()
        self._call("launch_count", C.byref(n))
        return n.value

    STAGES = ("triangle_test", "raster_setup_colour", "raster_setup_depth", "raster_bands", "resolve", "sort", "cull_bake", "triangle_compact")

    def frame_begin(self):
        self._call("frame_begin")

    def frame_end(self):
        self._call("frame_end")

    def frame_graph_stats(self):
        s = (C.c_uint64 * 4)()
        self._call("frame_graph_stats", s)
        return {"frames": int(s[0]), "graphed": int(s[1]), "flushed": int(s[2]), "instantiations": int(s[3])}

    def set_stage_timing(self, enabled: bool = True):
        self._call("set_stage_timing", C.c_int(1 if enabled else 0))

    def stage_times(self):
        ms, n = (C.c_double * 8)(), (C.c_uint32 * 8)()
        self._call("stage_times", ms, n)
        return {name: {"ms": float(ms[i]), "launches": int(n[i])} for i, name in enumerate(self.STAGES)}

    # ---- world data
    def set_objects(self, records: np.ndarray):
        records = np.ascontiguousarray(records)
        assert records.dtype.itemsize == 128
        self._call("set_objects", _ptr(records), C.c_uint32(len(records)))

    def set_objects_device(self, device_ptr: int, n_slots: int):
        self._call("set_objects_device", C.c_void_p(device_ptr), C.c_uint32(n_slots))

    def update_objects(self, slots: np.ndarray, records: np.ndarray):
        slots = np.ascontiguousarray(slots, dtype=np.uint32)
        records = np.ascontiguousarray(records)
        self._call("update_objects", _ptr(slots), _ptr(records), C.c_uint32(len(slots)))

    def set_object_sort_info(self, material_key, flags, location):
        k = np.ascontiguousarray(material_key, dtype=np.uint64)
        f = np.ascontiguousarray(flags, dtype=np.uint8)
        l = np.ascontiguousarray(location, dtype=np.float32).reshape(-1)
        assert len(f) == len(k) and len(l) == 3 * len(k)
        self._call("set_object_sort_info", _ptr(k), _ptr(f), _ptr(l), C.c_uint32(len(k)))

    def update_object_sort_info(self, slots, material_key, flags, location):
        s = np.ascontiguousarray(slots, dtype=np.uint32)
        k = np.ascontiguousarray(material_key, dtype=np.uint64)
        f = np.ascontiguousarray(flags, dtype=np.uint8)
        l = np.ascontiguousarray(location, dtype=np.float32).reshape(-1)
        assert len(k) == len(s) and len(f) == len(s) and len(l) == 3 * len(s)
        self._call("update_object_sort_info", _ptr(s), _ptr(k), _ptr(f), _ptr(l), C.c_uint32(len(s)))

    def resize_objects(self, n_slots: int):
        self._call("resize_objects", C.c_uint32(n_slots))

    # ---- objects that move (Renderer::set_object_transform in bulk)
    def set_object_mesh_spheres(self, spheres, slots=None):
        """(n, 4) mesh spheres (centre, radius) for slots 0 .. n-1, or for the listed slots."""
        sp = np.ascontiguousarray(spheres, dtype=np.float32).reshape(-1, 4)
        s = None if slots is None else np.ascontiguousarray(slots, dtype=np.uint32)
        assert s is None or len(s) == len(sp)
        self._call("set_object_mesh_spheres", _ptr(s), _ptr(sp) if len(sp) else None, C.c_uint32(len(sp)))

    def set_object_transforms(self, matrices, slots=None):
        """(n, 16) column-major matrices from host memory for slots 0 .. n-1, or for the listed slots.  Blocking."""
        m = np.ascontiguousarray(matrices, dtype=np.float32).reshape(-1, 16)
        s = None if slots is None else np.ascontiguousarray(slots, dtype=np.uint32)
        assert s is None or len(s) == len(m)
        self._call("set_object_transforms", _ptr(s), _ptr(m) if len(m) else None, C.c_uint32(len(m)))

    def set_object_transforms_device(self, matrices, slots=None, n: Optional[int] = None):
        """The same from device memory, enqueue only.  `matrices` / `slots` are CUDA tensors (contiguous float32 (n, 16) / int32 or uint32
        (n,)) or raw device pointers with `n` given; the caller keeps them alive and orders their producer on stream()."""
        def pointer(x, width):
            if x is None or isinstance(x, int):
                return x, None
            assert x.is_cuda and x.is_contiguous() and x.element_size() == 4, "a contiguous CUDA tensor of 4-byte elements"
            return x.data_ptr(), x.numel() // width
        mp, mn = pointer(matrices, 16)
        sp, sn = pointer(slots, 1)
        n = mn if n is None else n
        assert n is not None and (sn is None or sn == n)
        self._call("set_object_transforms_device", C.c_void_p(sp), C.c_void_p(mp), C.c_uint32(n))

    # ---- objects that come and go (ObjectManager::add into a prepared slot / remove)
    def set_objects_enabled(self, enabled, slots=None):
        """Slots 0 .. n-1, or the listed slots, present (enabled != 0) or absent, from host memory.  Blocking."""
        e = np.asarray(enabled)
        assert e.ndim == 1 and (e.dtype == np.bool_ or e.dtype == np.uint8), "enabled: a 1-d bool or uint8 array"
        e = np.ascontiguousarray(e).view(np.uint8)
        s = None
        if slots is not None:
            s = np.asarray(slots)
            assert s.ndim == 1 and s.dtype.kind in "iu" and len(s) == len(e), "slots: a 1-d integer array as long as enabled"
            assert not len(s) or (s.min() >= 0 and s.max() <= 0xFFFFFFFF), "slots: out of the uint32 range"
            s = np.ascontiguousarray(s, dtype=np.uint32)
        self._call("set_objects_enabled", _ptr(s), _ptr(e) if len(e) else None, C.c_uint32(len(e)))

    def set_objects_enabled_device(self, enabled, slots=None, n: Optional[int] = None):
        """The same from device memory, enqueue only.  `enabled` (bool / uint8 (n,)) and `slots` (int32 / uint32 (n,), None: slots
        0 .. n-1) are contiguous CUDA tensors, or raw device pointers with `n` given; the caller keeps them alive and orders their producer
        on stream()."""
        def pointer(x, sizes, what):
            if x is None or isinstance(x, int):
                return x, None
            assert getattr(x, "is_cuda", False) and x.is_contiguous() and x.dim() == 1 and x.element_size() in sizes \
                and not x.is_floating_point(), f"{what}: a contiguous 1-d CUDA tensor of {sizes[0]}-byte integers"
            return x.data_ptr(), x.numel()
        ep, en = pointer(enabled, (1,), "enabled")
        sp, sn = pointer(slots, (4,), "slots")
        n = en if n is None else n
        assert n is not None and (sn is None or sn == n) and (en is None or en == n), "enabled and slots differ in length"
        self._call("set_objects_enabled_device", C.c_void_p(sp), C.c_void_p(ep), C.c_uint32(n))

    def set_mesh_buffer(self, words: np.ndarray):
        words = np.ascontiguousarray(words, dtype=np.uint32)
        self._call("set_mesh_buffer", _ptr(words), C.c_uint64(words.nbytes))

    def update_mesh_buffer(self, byte_offset: int, data: np.ndarray):
        raw = np.ascontiguousarray(data).view(np.uint8).reshape(-1)
        self._call("update_mesh_buffer", C.c_uint64(byte_offset), _ptr(raw) if len(raw) else None, C.c_uint64(len(raw)))

    def update_textures(self, first: int, descs: np.ndarray, blob_offset: int, texels: np.ndarray):
        descs = np.ascontiguousarray(descs)
        texels = np.ascontiguousarray(texels).view(np.uint8).reshape(-1)
        assert descs.dtype.itemsize == 32
        self._call("update_textures", C.c_uint32(first), _ptr(descs) if len(descs) else None, C.c_uint32(len(descs)), C.c_uint64(blob_offset),
                   _ptr(texels) if len(texels) else None, C.c_uint64(len(texels)))

    def set_materials(self, records: np.ndarray):
        records = np.ascontiguousarray(records)
        assert records.dtype.itemsize == 208
        self._call("set_materials", _ptr(records), C.c_uint32(len(records)))

    # ---- materials that change (MaterialManager::update, evaluate's scatter of the stale records)
    def update_materials(self, records, indices=None):
        """Materials 0 .. n-1, or the listed indices, replaced by MATERIAL_DTYPE records from host memory; an index past the table's count
        grows it.  Blocking."""
        from .layouts import MATERIAL_DTYPE

        r = np.asarray(records)
        assert r.ndim == 1 and r.dtype == MATERIAL_DTYPE, "records: a 1-d MATERIAL_DTYPE array"
        r = np.ascontiguousarray(r)
        i = None
        if indices is not None:
            i = np.asarray(indices)
            assert i.ndim == 1 and i.dtype.kind in "iu" and len(i) == len(r), "indices: a 1-d integer array as long as records"
            assert not len(i) or (i.min() >= 0 and i.max() <= 0xFFFFFFFF), "indices: out of the uint32 range"
            i = np.ascontiguousarray(i, dtype=np.uint32)
        self._call("update_materials", _ptr(i), _ptr(r) if len(r) else None, C.c_uint32(len(r)))

    def update_materials_device(self, records, indices=None, n: Optional[int] = None):
        """The same from device memory, enqueue only; indices past the count are dropped.  `records` (uint8 (n, 208) or (n * 208,), or
        float32 / int32 / uint32 (n, 52): the 208-byte records, 16-byte aligned) and `indices` (int32 / uint32 (n,), None: materials
        0 .. n-1) are contiguous CUDA tensors, or raw device pointers with `n` given; the caller keeps them alive and orders their
        producer on stream()."""
        def pointer(x, what, ok, count):
            if x is None or isinstance(x, int):
                return x, None
            assert getattr(x, "is_cuda", False) and x.is_contiguous() and ok(x), what
            return x.data_ptr(), count(x)
        rp, rn = pointer(records, "records: a contiguous CUDA tensor of 208-byte rows (uint8 x 208 or 4-byte x 52), 16-byte aligned",
                         lambda x: x.numel() * x.element_size() % 208 == 0 and x.data_ptr() % 16 == 0
                         and (x.element_size() == 1 and not x.is_floating_point() or x.element_size() == 4)
                         and (x.dim() == 1 or x.dim() == 2 and x.shape[1] * x.element_size() == 208),
                         lambda x: x.numel() * x.element_size() // 208)
        ip, inn = pointer(indices, "indices: a contiguous 1-d CUDA tensor of 4-byte integers",
                          lambda x: x.dim() == 1 and x.element_size() == 4 and not x.is_floating_point(), lambda x: x.numel())
        n = rn if n is None else n
        assert n is not None and (inn is None or inn == n) and (rn is None or rn == n), "records and indices differ in length"
        self._call("update_materials_device", C.c_void_p(ip), C.c_void_p(rp), C.c_uint32(n))

    def readback_materials(self, first: int, n: int):
        """MATERIAL_DTYPE[n]: materials [first, first + n) of the table the shading reads.  Blocking."""
        from .layouts import MATERIAL_DTYPE

        out = np.zeros(max(n, 1), dtype=MATERIAL_DTYPE)
        self._call("readback_materials", _ptr(out), C.c_uint32(first), C.c_uint32(n))
        return out[:n]

    def set_textures(self, descs: np.ndarray, texels: np.ndarray):
        descs = np.ascontiguousarray(descs)
        texels = np.ascontiguousarray(texels).view(np.uint8).reshape(-1)
        assert descs.dtype.itemsize == 32
        self._call("set_textures", _ptr(descs) if len(descs) else None, C.c_uint32(len(descs)), _ptr(texels) if len(texels) else None, C.c_uint64(len(texels)))

    def set_skybox(self, desc: Optional[np.ndarray], texels: Optional[np.ndarray]):
        if desc is None:
            self._call("set_skybox", None, None, C.c_uint64(0))
            return
        desc = np.ascontiguousarray(desc).reshape(1)
        texels = np.ascontiguousarray(texels).view(np.uint8).reshape(-1)
        self._call("set_skybox", _ptr(desc), _ptr(texels), C.c_uint64(len(texels)))

    # ---- textures that change (rectangles of texels into the table's levels and the skybox's faces)
    def write_texture_regions(self, regions, texels):
        """TEXTURE_REGION_DTYPE regions (a contiguous 1-d array) copying bytes of `texels` (any contiguous host array, taken as its raw
        bytes) into the table's and the skybox's levels.  Checked as a whole first; blocking."""
        from .layouts import TEXTURE_REGION_DTYPE

        r = regions
        assert isinstance(r, np.ndarray) and r.dtype == TEXTURE_REGION_DTYPE and r.ndim == 1 and r.flags.c_contiguous, \
            "regions: a contiguous 1-d TEXTURE_REGION_DTYPE array"
        assert isinstance(texels, np.ndarray) and texels.flags.c_contiguous, "texels: a contiguous host array"
        t = texels.reshape(-1).view(np.uint8)
        self._call("write_texture_regions", _ptr(r) if len(r) else None, C.c_uint32(len(r)), _ptr(t) if len(t) else None, C.c_uint64(len(t)))

    def write_texture_regions_device(self, regions, texels, n: Optional[int] = None):
        """The same from device memory, enqueue only; invalid regions are dropped.  `regions` is a contiguous CUDA tensor of 40-byte records
        (uint8 (n, 40), int32 / uint32 (n, 10) or int64 / uint64 (n, 5)) at an 8-byte aligned address, `texels` a contiguous CUDA tensor
        taken as its raw bytes; `n` (default: every row) may name fewer regions.  The caller keeps both alive and orders their producer on
        stream()."""
        x = regions
        assert getattr(x, "is_cuda", False) and x.is_contiguous() and x.dim() == 2 and x.element_size() in (1, 4, 8) \
            and x.shape[1] * x.element_size() == 40 and not x.is_floating_point() and x.data_ptr() % 8 == 0, \
            "regions: a contiguous, 8-byte aligned CUDA tensor of 40-byte integer rows"
        assert getattr(texels, "is_cuda", False) and texels.is_contiguous(), "texels: a contiguous CUDA tensor"
        n = x.shape[0] if n is None else n
        assert 0 <= n <= x.shape[0], "n: at most the regions' row count"
        nbytes = texels.numel() * texels.element_size()
        self._call("write_texture_regions_device", C.c_void_p(x.data_ptr()), C.c_uint32(n), C.c_void_p(texels.data_ptr() if nbytes else None),
                   C.c_uint64(nbytes))

    def readback_texels(self, skybox: bool, byte_offset: int, nbytes: int) -> np.ndarray:
        """nbytes of the table's blob (skybox False) or the skybox's, from byte_offset, as uint8.  Blocking."""
        out = np.zeros(max(nbytes, 1), dtype=np.uint8)
        self._call("readback_texels", C.c_int(1 if skybox else 0), C.c_uint64(byte_offset), _ptr(out), C.c_uint64(nbytes))
        return out[:nbytes]

    def set_directional_lights(self, data: bytes, atlas_w: int, atlas_h: int):
        self._call("set_directional_lights", C.c_char_p(data), C.c_uint64(len(data)), C.c_uint32(atlas_w), C.c_uint32(atlas_h))

    # ---- directional lights evaluated on the device (rule R13)
    def set_directional_light_sources(self, sources: np.ndarray, atlas_w: int, atlas_h: int, left_handed: bool):
        from .layouts import LIGHT_SOURCE_DTYPE

        src = np.ascontiguousarray(sources, dtype=LIGHT_SOURCE_DTYPE).reshape(-1)
        self._call("set_directional_light_sources", _ptr(src) if len(src) else None, C.c_uint32(len(src)), C.c_uint32(atlas_w),
                   C.c_uint32(atlas_h), C.c_uint32(1 if left_handed else 0))

    def evaluate_shadow_cameras(self, viewport_location):
        loc = np.ascontiguousarray(viewport_location, dtype=np.float32).reshape(3)
        self._call("evaluate_shadow_cameras", _ptr(loc))

    def shadow_uniform_upload(self, shadow_index: int, object_count: int, mode: int = CB_BAKE | CB_CULL):
        self._call("shadow_uniform_upload", C.c_uint32(shadow_index), C.c_uint32(object_count), C.c_uint32(mode))

    def update_directional_light_sources(self, changes):
        """DirectionalLightChanges from host memory: a contiguous 1-d DIRECTIONAL_LIGHT_CHANGE_DTYPE array.  Enqueue only."""
        from .layouts import DIRECTIONAL_LIGHT_CHANGE_DTYPE

        c = changes
        assert isinstance(c, np.ndarray) and c.dtype == DIRECTIONAL_LIGHT_CHANGE_DTYPE and c.ndim == 1 and c.flags.c_contiguous, \
            "changes: a contiguous 1-d DIRECTIONAL_LIGHT_CHANGE_DTYPE array"
        self._call("update_directional_light_sources", _ptr(c) if len(c) else None, C.c_uint32(len(c)))

    def update_directional_light_sources_device(self, changes, n: Optional[int] = None):
        """The same from device memory, enqueue only; entries naming no light or carrying an unknown mask bit are dropped.  `changes` is
        a contiguous CUDA tensor of 48-byte records (uint8 (n, 48), or int32 / uint32 / float32 (n, 12)), or a raw device pointer with `n`
        given; the caller keeps it alive and orders its producer on stream()."""
        if isinstance(changes, int):
            assert n is not None, "changes: a raw pointer needs n"
            ptr = changes
        else:
            x = changes
            assert getattr(x, "is_cuda", False) and x.is_contiguous() and x.dim() == 2 and x.element_size() in (1, 4) \
                and x.shape[1] * x.element_size() == 48 and not (x.element_size() == 1 and x.is_floating_point()) \
                and x.data_ptr() % 4 == 0, "changes: a contiguous CUDA tensor of 48-byte records (uint8 (n, 48) or 4-byte (n, 12))"
            assert n is None or n == x.shape[0], "n: the tensor's row count"
            ptr, n = x.data_ptr(), x.shape[0]
        self._call("update_directional_light_sources_device", C.c_void_p(ptr), C.c_uint32(n))

    def readback_shadow_cameras(self, n: int):
        """(CAMERA_HEADER_DTYPE[n], DIRECTIONAL_LIGHT_DTYPE[n])"""
        from .layouts import DIRECTIONAL_LIGHT_DTYPE

        heads = np.zeros(max(n, 1), dtype=CAMERA_HEADER_DTYPE)
        lights = np.zeros(max(n, 1), dtype=DIRECTIONAL_LIGHT_DTYPE)
        self._call("readback_shadow_cameras", _ptr(heads), _ptr(lights), C.c_uint32(n))
        return heads[:n], lights[:n]

    def set_point_lights(self, data: bytes):
        self._call("set_point_lights", C.c_char_p(data), C.c_uint64(len(data)))

    # ---- PointLightManager on the device (handle table, add / update / remove, evaluate)
    def set_point_light_sources(self, sources: np.ndarray, live: Optional[np.ndarray] = None):
        """The whole handle table: POINT_LIGHT_SOURCE_DTYPE[n] and live bytes (None: every handle live).  Blocking."""
        from .layouts import POINT_LIGHT_SOURCE_DTYPE

        src = np.ascontiguousarray(sources, dtype=POINT_LIGHT_SOURCE_DTYPE).reshape(-1)
        lv = None if live is None else np.ascontiguousarray(live, dtype=np.uint8).reshape(-1)
        assert lv is None or len(lv) == len(src)
        self._call("set_point_light_sources", _ptr(src) if len(src) else None, _ptr(lv) if lv is not None and len(lv) else None, C.c_uint32(len(src)))

    def update_point_light_sources(self, handles, sources: np.ndarray, live):
        """add / update (live != 0) or remove (live == 0) of the listed handles, from host memory.  Blocking."""
        from .layouts import POINT_LIGHT_SOURCE_DTYPE

        h = np.ascontiguousarray(handles, dtype=np.uint32).reshape(-1)
        src = np.ascontiguousarray(sources, dtype=POINT_LIGHT_SOURCE_DTYPE).reshape(-1)
        lv = np.ascontiguousarray(live, dtype=np.uint8).reshape(-1)
        assert len(src) == len(h) and len(lv) == len(h)
        self._call("update_point_light_sources", _ptr(h), _ptr(src), _ptr(lv), C.c_uint32(len(h)))

    def update_point_light_sources_device(self, handles, sources, live=None, n: Optional[int] = None):
        """The same from device memory, enqueue only.  `handles` (int32 / uint32 (n,)), `sources` (float32 (n, 8): the 32-byte records)
        and `live` (uint8 (n,), None: every handle live) are contiguous CUDA tensors, or raw device pointers with `n` given; the caller
        keeps them alive and orders their producer on stream()."""
        def pointer(x, elem, width):
            if x is None or isinstance(x, int):
                return x, None
            assert x.is_cuda and x.is_contiguous() and x.element_size() == elem, "a contiguous CUDA tensor"
            return x.data_ptr(), x.numel() // width
        hp, hn = pointer(handles, 4, 1)
        sp, sn = pointer(sources, 4, 8)
        lp, ln = pointer(live, 1, 1)
        n = hn if n is None else n
        assert n is not None and (sn is None or sn == n) and (ln is None or ln == n)
        self._call("update_point_light_sources_device", C.c_void_p(hp), C.c_void_p(sp), C.c_void_p(lp), C.c_uint32(n))

    def evaluate_point_lights(self):
        self._call("evaluate_point_lights")

    def readback_point_lights(self) -> bytes:
        """The buffer the shading reads: u32 count @0, POINT_LIGHT_DTYPE array @16 (as EvalOutput.point_buffer)."""
        head = np.zeros(4, dtype=np.uint32)
        self._call("readback_point_lights", _ptr(head), C.c_uint64(16))
        out = np.zeros(16 + 32 * int(head[0]), dtype=np.uint8)
        self._call("readback_point_lights", _ptr(out), C.c_uint64(len(out)))
        return out.tobytes()

    def set_frame_uniforms(self, record: np.ndarray):
        b = record.tobytes()
        assert len(b) == 496
        self._call("set_frame_uniforms", C.c_char_p(b))

    # ---- skinning
    def skin(self, inputs: np.ndarray, joint_matrices: np.ndarray):
        inputs = np.ascontiguousarray(inputs)
        assert inputs.dtype.itemsize == 40
        jm = np.ascontiguousarray(joint_matrices, dtype=np.float32).reshape(-1, 16)
        self._call("skin", _ptr(inputs), C.c_uint32(len(inputs)), _ptr(jm), C.c_uint32(len(jm)))

    def readback_mesh_buffer(self, n_words: int) -> np.ndarray:
        out = np.empty(n_words, dtype=np.uint32)
        self._call("readback_mesh_buffer", _ptr(out), C.c_uint64(out.nbytes))
        return out

    # ---- skeletal animation (posed on the device, skinned from resident joint matrices)
    def set_animations(self, skins: np.ndarray, joints: np.ndarray, order: np.ndarray, clips: np.ndarray, channels: np.ndarray, keys: np.ndarray):
        arrays = [np.ascontiguousarray(skins), np.ascontiguousarray(joints), np.ascontiguousarray(order, dtype=np.uint32),
                  np.ascontiguousarray(clips), np.ascontiguousarray(channels), np.ascontiguousarray(keys, dtype=np.float32)]
        s, j, o, c, ch, k = arrays
        assert (s.dtype.itemsize, j.dtype.itemsize, c.dtype.itemsize, ch.dtype.itemsize) == (8, 112, 16, 64) and len(o) == len(j)
        lib = _AnimLibrary(_ptr(s) if len(s) else None, len(s), _ptr(j) if len(j) else None, len(j), _ptr(o) if len(o) else None,
                           _ptr(c) if len(c) else None, len(c), _ptr(ch) if len(ch) else None, len(ch), _ptr(k) if len(k) else None, len(k))
        self._call("set_animations", C.byref(lib))

    def set_skeletons(self, inputs: np.ndarray, joint_matrices: np.ndarray):
        inputs = np.ascontiguousarray(inputs)
        assert inputs.dtype.itemsize == 40
        jm = np.ascontiguousarray(joint_matrices, dtype=np.float32).reshape(-1, 16)
        self._call("set_skeletons", _ptr(inputs) if len(inputs) else None, C.c_uint32(len(inputs)), _ptr(jm) if len(jm) else None, C.c_uint32(len(jm)))

    def set_pose_jobs(self, jobs: np.ndarray, targets: np.ndarray):
        jobs, targets = np.ascontiguousarray(jobs), np.ascontiguousarray(targets)
        assert jobs.dtype.itemsize == 16 and targets.dtype.itemsize == 8
        self._call("set_pose_jobs", _ptr(jobs) if len(jobs) else None, C.c_uint32(len(jobs)), _ptr(targets) if len(targets) else None, C.c_uint32(len(targets)))

    def pose_skeletons(self):
        self._call("pose_skeletons")

    def skin_posed(self):
        self._call("skin_posed")

    def readback_joint_matrices(self, first: int, n: int) -> np.ndarray:
        out = np.empty((max(n, 1), 16), dtype=np.float32)
        self._call("readback_joint_matrices", _ptr(out), C.c_uint32(first), C.c_uint32(n))
        return out[:n]

    # ---- joint matrices set by the application (Renderer::set_skeleton_joint_matrices / set_skeleton_joint_transforms)
    def set_joint_matrices(self, writes, mat4s, inverse_binds=None):
        """JOINT_WRITE_DTYPE writes into the joint buffer from host memory: mat4s ((m, 16) or (m, 4, 4) float32, column-major) copied bit
        for bit, or times `inverse_binds` (the same shapes) when given.  Blocking."""
        from .layouts import JOINT_WRITE_DTYPE

        w = np.asarray(writes)
        assert w.ndim == 1 and w.dtype == JOINT_WRITE_DTYPE, "writes: a 1-d JOINT_WRITE_DTYPE array"
        w = np.ascontiguousarray(w)

        def mats(x, what):
            x = np.asarray(x)
            assert x.dtype == np.float32 and x.ndim in (2, 3) and x.shape[1:] in ((16,), (4, 4)), f"{what}: float32 (m, 16) or (m, 4, 4)"
            return np.ascontiguousarray(x).reshape(-1, 16)
        m = mats(mat4s, "mat4s")
        ib = None if inverse_binds is None else mats(inverse_binds, "inverse_binds")
        # an empty inverse-bind array still passes a pointer: null selects the copy form
        self._call("set_joint_matrices", _ptr(w), C.c_uint32(len(w)), _ptr(m), C.c_uint32(len(m)), _ptr(ib), C.c_uint32(0 if ib is None else len(ib)))

    def set_joint_matrices_device(self, writes, mat4s, inverse_binds=None, n_writes: Optional[int] = None, n_mat4s: Optional[int] = None,
                                  n_inverse_binds: Optional[int] = None):
        """The same from device memory, enqueue only; writes outside their arrays or the joint buffer are dropped whole.  `writes` (uint8
        (n, 16) / (n * 16,), or int32 / uint32 (n, 4): JOINT_WRITE_DTYPE records), `mat4s` and `inverse_binds` (float32 (m, 16) or
        (m, 4, 4), 16-byte aligned) are contiguous CUDA tensors, or raw device pointers with their count given; the caller keeps them alive
        and orders their producer on stream()."""
        def pointer(x, count, what, ok, rows):
            if x is None or isinstance(x, int):
                assert x is None or count is not None, f"{what}: a raw pointer needs its count"
                return x, (0 if x is None else count)
            assert getattr(x, "is_cuda", False) and x.is_contiguous() and ok(x), what
            return x.data_ptr(), rows(x)
        wp, wn = pointer(writes, n_writes, "writes: a contiguous CUDA tensor of 16-byte JOINT_WRITE records (uint8 x 16 or 4-byte integers x 4)",
                         lambda x: not x.is_floating_point() and x.element_size() in (1, 4) and x.numel() * x.element_size() % 16 == 0
                         and (x.dim() == 1 or x.dim() == 2 and x.shape[1] * x.element_size() == 16),
                         lambda x: x.numel() * x.element_size() // 16)
        mat_ok = lambda x: (str(x.dtype) == "torch.float32" and x.data_ptr() % 16 == 0 and x.dim() in (2, 3)
                            and tuple(x.shape[1:]) in ((16,), (4, 4)))
        mp, mn = pointer(mat4s, n_mat4s, "mat4s: a contiguous float32 CUDA tensor (m, 16) or (m, 4, 4), 16-byte aligned", mat_ok, lambda x: x.shape[0])
        ip, inn = pointer(inverse_binds, n_inverse_binds, "inverse_binds: a contiguous float32 CUDA tensor (m, 16) or (m, 4, 4), 16-byte aligned",
                          mat_ok, lambda x: x.shape[0])
        self._call("set_joint_matrices_device", C.c_void_p(wp), C.c_uint32(wn), C.c_void_p(mp), C.c_uint32(mn), C.c_void_p(ip), C.c_uint32(inn))

    # ---- meshes that deform every frame (rebuild of the mesh + re-add of its objects, on the device)
    def set_deformable_meshes(self, meshes, object_slots=None, object_meshes=None):
        """DEFORMABLE_MESH_DTYPE records and the (slot, mesh) pairs of the objects that draw them.  Blocking."""
        from .layouts import DEFORMABLE_MESH_DTYPE

        m = np.asarray(meshes)
        assert m.ndim == 1 and m.dtype == DEFORMABLE_MESH_DTYPE, "meshes: a 1-d DEFORMABLE_MESH_DTYPE array"
        m = np.ascontiguousarray(m)
        s = np.ascontiguousarray(np.zeros(0) if object_slots is None else object_slots, dtype=np.uint32).reshape(-1)
        o = np.ascontiguousarray(np.zeros(0) if object_meshes is None else object_meshes, dtype=np.uint32).reshape(-1)
        assert len(s) == len(o), "object_slots and object_meshes: one mesh per slot"
        self._call("set_deformable_meshes", _ptr(m) if len(m) else None, C.c_uint32(len(m)), _ptr(s) if len(s) else None,
                   _ptr(o) if len(o) else None, C.c_uint32(len(s)))

    def deform_meshes(self, positions):
        """New positions of every mesh of the set from host memory: float32 (sum(vertex_count), 3), mesh after mesh.  Blocking."""
        p = np.asarray(positions)
        assert p.dtype == np.float32 and p.ndim == 2 and p.shape[1] == 3, "positions: float32 (n, 3)"
        p = np.ascontiguousarray(p)
        self._call("deform_meshes", _ptr(p) if p.size else None, C.c_uint64(p.size))

    def deform_meshes_device(self, positions, n_floats: Optional[int] = None):
        """The same from device memory, enqueue only: a contiguous float32 CUDA tensor (n, 3), or a raw device pointer with n_floats
        given; the caller keeps it alive and orders its producer on stream()."""
        if isinstance(positions, int):
            assert n_floats is not None, "positions: a raw pointer needs n_floats"
            ptr, n = positions, n_floats
        else:
            assert getattr(positions, "is_cuda", False) and positions.is_contiguous() and str(positions.dtype) == "torch.float32" \
                and positions.dim() == 2 and positions.shape[1] == 3 and positions.data_ptr() % 4 == 0, \
                "positions: a contiguous float32 CUDA tensor (n, 3)"
            ptr, n = positions.data_ptr(), positions.numel()
        self._call("deform_meshes_device", C.c_void_p(ptr), C.c_uint64(n))

    def readback_deformable_mesh_spheres(self, first: int, n: int) -> np.ndarray:
        """(n, 4) mesh spheres (centre, radius) of the set's meshes [first, first + n) from the last deform"""
        out = np.zeros((max(n, 1), 4), dtype=np.float32)
        self._call("readback_deformable_mesh_spheres", _ptr(out), C.c_uint32(first), C.c_uint32(n))
        return out[:n]

    # ---- objects that change mesh or material (ObjectManager::add with another mesh kind or material)
    def set_object_variants(self, variants, groups, slots=None, slot_groups=None):
        """OBJECT_VARIANT_DTYPE records, VARIANT_GROUP_DTYPE groups (runs of variants) and the (slot, group) pairs of the listed slots.
        Blocking; an empty `variants` removes the set."""
        from .layouts import OBJECT_VARIANT_DTYPE, VARIANT_GROUP_DTYPE

        v, g = np.asarray(variants), np.asarray(groups)
        assert v.ndim == 1 and v.dtype == OBJECT_VARIANT_DTYPE, "variants: a 1-d OBJECT_VARIANT_DTYPE array"
        assert g.ndim == 1 and g.dtype == VARIANT_GROUP_DTYPE, "groups: a 1-d VARIANT_GROUP_DTYPE array"
        s = _u32_list(np.zeros(0, np.uint32) if slots is None else slots, "slots")
        sg = _u32_list(np.zeros(0, np.uint32) if slot_groups is None else slot_groups, "slot_groups")
        assert len(s) == len(sg), "slots and slot_groups: one group per slot"
        v, g = np.ascontiguousarray(v), np.ascontiguousarray(g)
        self._call("set_object_variants", _ptr(v) if len(v) else None, C.c_uint32(len(v)), _ptr(g) if len(g) else None, C.c_uint32(len(g)),
                   _ptr(s) if len(s) else None, _ptr(sg) if len(sg) else None, C.c_uint32(len(s)))

    def switch_object_variants(self, choices, slots=None):
        """Slots 0 .. n-1, or the listed slots, to variant group.first + choices[i] of their group, from host memory.  Blocking."""
        c = _u32_list(choices, "choices")
        s = None if slots is None else _u32_list(slots, "slots")
        assert s is None or len(s) == len(c), "slots: as long as choices"
        self._call("switch_object_variants", _ptr(s) if s is not None and len(s) else None, _ptr(c) if len(c) else None, C.c_uint32(len(c)))

    def switch_object_variants_device(self, choices, slots=None, n: Optional[int] = None):
        """The same from device memory, enqueue only.  `choices` and `slots` (None: slots 0 .. n-1) are contiguous 1-d CUDA tensors of
        4-byte integers, or raw device pointers with `n` given; the caller keeps them alive and orders their producer on stream()."""
        def pointer(x, what):
            if x is None or isinstance(x, int):
                return x, None
            assert getattr(x, "is_cuda", False) and x.is_contiguous() and x.dim() == 1 and x.element_size() == 4 \
                and not x.is_floating_point(), f"{what}: a contiguous 1-d CUDA tensor of 4-byte integers"
            return x.data_ptr(), x.numel()
        cp, cn = pointer(choices, "choices")
        sp, sn = pointer(slots, "slots")
        n = cn if n is None else n
        assert n is not None and (sn is None or sn == n) and (cn is None or cn == n), "choices and slots differ in length"
        self._call("switch_object_variants_device", C.c_void_p(sp), C.c_void_p(cp), C.c_uint32(n))

    def readback_object_variants(self, first: int, n: int) -> np.ndarray:
        """The current variant of slots [first, first + n): an index into the table, VARIANT_NONE when unlisted or never switched"""
        out = np.zeros(max(n, 1), dtype=np.uint32)
        self._call("readback_object_variants", _ptr(out), C.c_uint32(first), C.c_uint32(n))
        return out[:n]

    # ---- meshes whose topology changes every frame (rebuild of the mesh from new vertices and indices + re-add of its objects, on the device)
    def set_remeshable_meshes(self, meshes, object_slots=None, object_meshes=None):
        """REMESHABLE_MESH_DTYPE records and the (slot, mesh) pairs of the objects that draw them.  Blocking."""
        from .layouts import REMESHABLE_MESH_DTYPE

        m = np.asarray(meshes)
        assert m.ndim == 1 and m.dtype == REMESHABLE_MESH_DTYPE, "meshes: a 1-d REMESHABLE_MESH_DTYPE array"
        m = np.ascontiguousarray(m)
        s = np.ascontiguousarray(np.zeros(0) if object_slots is None else object_slots, dtype=np.uint32).reshape(-1)
        o = np.ascontiguousarray(np.zeros(0) if object_meshes is None else object_meshes, dtype=np.uint32).reshape(-1)
        assert len(s) == len(o), "object_slots and object_meshes: one mesh per slot"
        self._call("set_remeshable_meshes", _ptr(m) if len(m) else None, C.c_uint32(len(m)), _ptr(s) if len(s) else None,
                   _ptr(o) if len(o) else None, C.c_uint32(len(s)))

    _REMESH_STREAMS = (("counts", "uint32", 2), ("positions", "float32", 3), ("indices", "uint32", None), ("normals", "float32", 3),
                       ("tangents", "float32", 3), ("uv0", "float32", 2), ("color0", "uint32", None))

    @staticmethod
    def _remesh_arrays(arrays, dtype_of, is_ok):
        """checks each stream's shape and dtype: counts (n_meshes, 2) uint32, positions / normals / tangents (n_vertices, 3) float32, uv0
        (n_vertices, 2) float32, indices and color0 1-d uint32 (color0 one packed word per vertex); int32 is taken for uint32 (a negative
        value fails validation); returns (n_vertices, n_indices)"""
        n_v = n_i = None
        for (name, dt, cols), a in zip(Backend._REMESH_STREAMS, arrays):
            if a is None:
                assert name not in ("counts", "positions", "indices"), f"{name}: required"
                continue
            shape = tuple(a.shape)
            assert is_ok(a) and dtype_of(a) in ((dt, "int32") if dt == "uint32" else (dt,)) and (len(shape) == 1 if cols is None else (len(shape) == 2 and shape[1] == cols)), \
                f"{name}: a contiguous {dt} array of shape {'(n,)' if cols is None else f'(n, {cols})'}"
            if name == "indices":
                n_i = shape[0]
            elif name != "counts":
                assert n_v is None or n_v == shape[0], f"{name}: one row per vertex, as positions"
                n_v = shape[0]
        return n_v, n_i

    def remesh_meshes(self, counts, positions, indices, normals=None, tangents=None, uv0=None, color0=None):
        """New counts, vertices and indices of every mesh of the set from host memory, at capacity strides (see r3_remesh_meshes).
        Blocking; R3_E_INVALID, nothing written, when a mesh fails Mesh::validate."""
        arrays = [None if a is None else np.ascontiguousarray(a) for a in (counts, positions, indices, normals, tangents, uv0, color0)]
        n_v, n_i = self._remesh_arrays(arrays, lambda a: str(a.dtype), lambda a: True)
        self._call("remesh_meshes", *[None if a is None or a.size == 0 else _ptr(a) for a in arrays], C.c_uint64(n_v), C.c_uint64(n_i))

    def remesh_meshes_device(self, counts, positions, indices, normals=None, tangents=None, uv0=None, color0=None):
        """The same from device memory, enqueue only: contiguous CUDA tensors (4-byte aligned) of the host form's shapes and dtypes; the
        caller keeps them alive and orders their producer on stream().  A mesh that fails Mesh::validate is left as it was and reported
        by readback_remesh_status."""
        arrays = (counts, positions, indices, normals, tangents, uv0, color0)
        n_v, n_i = self._remesh_arrays(arrays, lambda a: str(a.dtype).replace("torch.", ""),
                                       lambda a: getattr(a, "is_cuda", False) and a.is_contiguous() and a.data_ptr() % 4 == 0)
        self._call("remesh_meshes_device", *[C.c_void_p(None if a is None else a.data_ptr()) for a in arrays], C.c_uint64(n_v), C.c_uint64(n_i))

    def readback_remesh_status(self, first: int, n: int):
        """(status (n,) uint32: REMESH_* of the last remesh, counts (n, 2) uint32: the {vertex_count, index_count} in force)"""
        status, counts = np.zeros(max(n, 1), np.uint32), np.zeros((max(n, 1), 2), np.uint32)
        self._call("readback_remesh_status", _ptr(status), _ptr(counts), C.c_uint32(first), C.c_uint32(n))
        return status[:n], counts[:n]

    def debug_invocation_bound(self):
        """Test hook: (sum, largest) of the per-slot invocation terms the culling buffers are sized with"""
        out = (C.c_uint64 * 2)()
        self._call("debug_invocation_bound", out)
        return int(out[0]), int(out[1])

    # ---- object animation (the object-transform half of pose_animation_frame, posed on the device)
    def set_object_animations(self, nodes: np.ndarray, clips: np.ndarray, channels: np.ndarray, keys: np.ndarray, left_handed: bool):
        n, c, ch = np.ascontiguousarray(nodes), np.ascontiguousarray(clips), np.ascontiguousarray(channels)
        k = np.ascontiguousarray(keys, dtype=np.float32)
        assert (n.dtype.itemsize, c.dtype.itemsize, ch.dtype.itemsize) == (48, 16, 64)
        lib = _AnimObjectLibrary(_ptr(n) if len(n) else None, len(n), _ptr(c) if len(c) else None, len(c), _ptr(ch) if len(ch) else None, len(ch),
                                 _ptr(k) if len(k) else None, len(k), 1 if left_handed else 0)
        self._call("set_object_animations", C.byref(lib))

    def set_object_pose_jobs(self, jobs: np.ndarray, targets: np.ndarray):
        jobs, targets = np.ascontiguousarray(jobs), np.ascontiguousarray(targets)
        assert jobs.dtype.itemsize == 16 and targets.dtype.itemsize == 32
        self._call("set_object_pose_jobs", _ptr(jobs) if len(jobs) else None, C.c_uint32(len(jobs)), _ptr(targets) if len(targets) else None,
                   C.c_uint32(len(targets)))

    def pose_objects(self):
        self._call("pose_objects")

    def readback_objects(self, first: int, n: int, locations: bool = True):
        """(records, (n, 3) sort locations or None)"""
        from .layouts import OBJECT_DTYPE

        out = np.zeros(max(n, 1), dtype=OBJECT_DTYPE)
        loc = np.zeros((max(n, 1), 3), dtype=np.float32) if locations else None
        self._call("readback_objects", _ptr(out), _ptr(loc), C.c_uint32(first), C.c_uint32(n))
        return out[:n], (loc[:n] if locations else None)

    # ---- object cull + bake
    def object_uniform_upload(self, camera: int, header: np.ndarray, mode: int = CB_BAKE | CB_CULL):
        b = header.tobytes()
        assert len(b) == CAMERA_HEADER_DTYPE.itemsize
        self._call("object_uniform_upload", C.c_uint32(camera), C.c_char_p(b), C.c_uint32(mode))

    def visible_count(self, camera: int) -> int:
        n = C.c_uint32()
        self._call("visible_count", C.c_uint32(camera), C.byref(n))
        return n.value

    def readback_visible(self, camera: int) -> np.ndarray:
        n = self.visible_count(camera)
        out = np.empty(max(n, 1), dtype=np.uint32)
        cnt = C.c_uint32()
        self._call("readback_visible", C.c_uint32(camera), _ptr(out), C.c_uint32(len(out)), C.byref(cnt))
        return out[: cnt.value]

    def readback_object_matrices(self, camera: int, first: int, n: int) -> np.ndarray:
        out = np.empty(max(n, 1), dtype=OBJECT_MATRICES_DTYPE)
        self._call("readback_object_matrices", C.c_uint32(camera), _ptr(out), C.c_uint32(first), C.c_uint32(n))
        return out[:n]

    # ---- batching + triangle cull
    def batch_objects(self, camera: int, viewport_location, max_dispatch_count: int = 65535):
        loc = np.ascontiguousarray(viewport_location, dtype=np.float32)
        self._call("batch_objects", C.c_uint32(camera), _ptr(loc), C.c_uint32(max_dispatch_count))

    def batch_counts(self, camera: int):
        a, b, c = C.c_uint32(), C.c_uint32(), C.c_uint32()
        self._call("batch_counts", C.c_uint32(camera), C.byref(a), C.byref(b), C.byref(c))
        return a.value, b.value, c.value

    def readback_batches(self, camera: int):
        nb, nr, _ = self.batch_counts(camera)
        batches = np.zeros(max(nb, 1), dtype=BATCH_DTYPE)
        regions = np.zeros(max(nr, 1), dtype=REGION_DTYPE)
        self._call("readback_batches", C.c_uint32(camera), _ptr(batches), _ptr(regions))
        return batches[:nb], regions[:nr]

    def batching_info(self, camera: int):
        info = (C.c_uint32 * 4)()
        self._call("batching_info", C.c_uint32(camera), info)
        return {"path": {0: "none", 1: "device", 2: "host", 3: "device, frame-wide sort"}[info[0]], "overflow": int(info[1]), "batches": int(info[2]), "regions": int(info[3])}

    def cull(self, camera: int, batches: Optional[np.ndarray] = None, regions: Optional[np.ndarray] = None):
        if batches is None:
            self._call("cull", C.c_uint32(camera), None, C.c_uint32(0), None, C.c_uint32(0))
        else:
            batches, regions = np.ascontiguousarray(batches), np.ascontiguousarray(regions)
            self._call("cull", C.c_uint32(camera), _ptr(batches), C.c_uint32(len(batches)), _ptr(regions), C.c_uint32(len(regions)))

    def _readback_counted(self, name, camera, partition, dtype, count_type=C.c_uint64):
        n = count_type()
        self._call(name, C.c_uint32(camera), C.c_int(partition), None, count_type(0), C.byref(n))
        out = np.empty(max(n.value, 1), dtype=dtype)
        self._call(name, C.c_uint32(camera), C.c_int(partition), _ptr(out), count_type(len(out)), C.byref(n))
        return out[: n.value]

    def readback_indices(self, camera: int, partition: int) -> np.ndarray:
        return self._readback_counted("readback_indices", camera, partition, np.uint32)

    def readback_draw_calls(self, camera: int, partition: int) -> np.ndarray:
        return self._readback_counted("readback_draw_calls", camera, partition, INDIRECT_CALL_DTYPE, C.c_uint32)

    def readback_culling_results(self, camera: int, partition: int) -> np.ndarray:
        return self._readback_counted("readback_culling_results", camera, partition, np.uint32)

    # ---- forward
    def set_render_target(self, width: int, height: int, samples: int = 1, clear=(0, 0, 0, 0)):
        c = (C.c_float * 4)(*[float(v) for v in clear])
        self._call("set_render_target", C.c_uint32(width), C.c_uint32(height), C.c_uint32(samples), c)
        self.width, self.height = width, height

    def set_scissor_rows(self, begin: int, end: int):
        self._call("set_scissor_rows", C.c_uint32(begin), C.c_uint32(end))

    def clear_shadow_atlas(self):
        self._call("clear_shadow_atlas")

    def shadow_pass(self, index: int, ox: int, oy: int, size: int):
        self._call("shadow_pass", C.c_uint32(index), C.c_uint32(ox), C.c_uint32(oy), C.c_uint32(size))

    def forward_begin(self):
        self._call("forward_begin")

    def forward_pass(self, source: int):
        self._call("forward_pass", C.c_int(source))

    def hiz_build(self):
        self._call("hiz_build")

    def forward_resolve(self):
        self._call("forward_resolve")

    # ---- multi-GPU exchange of the visible set over NVLink peer memory
    def exchange_create(self, camera: int, n_ranks: int, my_rank: int, max_objects_per_rank: int) -> bytes:
        h = (C.c_uint8 * 64)()
        self._call("exchange_create", C.c_uint32(camera), C.c_uint32(n_ranks), C.c_uint32(my_rank), C.c_uint32(max_objects_per_rank), h)
        return bytes(h)

    def exchange_connect(self, camera: int, handles: bytes):
        buf = (C.c_uint8 * len(handles)).from_buffer_copy(handles)
        self._call("exchange_connect", C.c_uint32(camera), buf)

    def exchange_words(self, camera: int):
        p, n, w = C.c_void_p(), C.c_uint64(), C.c_uint32()
        self._call("exchange_words", C.c_uint32(camera), C.byref(p), C.byref(n), C.byref(w))
        return p.value, n.value, w.value

    def exchange_merge(self, camera: int, rank_objects, rank_base=None):
        ro = np.ascontiguousarray(rank_objects, dtype=np.uint32)
        rb = None if rank_base is None else np.ascontiguousarray(rank_base, dtype=np.uint32)
        self._call("exchange_merge", C.c_uint32(camera), _ptr(ro), _ptr(rb))

    def exchange_count(self, camera: int, rank_objects):
        ro = np.ascontiguousarray(rank_objects, dtype=np.uint32)
        self._call("exchange_count", C.c_uint32(camera), _ptr(ro))

    def exchange_counts(self, camera: int, n_ranks: int) -> np.ndarray:
        out = np.zeros(n_ranks + 1, dtype=np.uint32)
        self._call("exchange_counts", C.c_uint32(camera), _ptr(out))
        return out

    def exchange_merged(self, camera: int):
        lst, cnt, cap = C.c_void_p(), C.c_void_p(), C.c_uint64()
        self._call("exchange_merged", C.c_uint32(camera), C.byref(lst), C.byref(cnt), C.byref(cap))
        return lst.value, cnt.value, cap.value

    def exchange_destroy(self, camera: int):
        self._call("exchange_destroy", C.c_uint32(camera))

    # ---- peer-memory plumbing of the multi-GPU forward pass
    def peer_create(self, n_ranks: int, my_rank: int) -> bytes:
        h = (C.c_uint8 * 256)()
        self._call("peer_create", C.c_uint32(n_ranks), C.c_uint32(my_rank), h)
        return bytes(h)

    def peer_connect(self, handles: bytes):
        buf = (C.c_uint8 * len(handles)).from_buffer_copy(handles)
        self._call("peer_connect", buf)

    def peer_send_atlas_rect(self, ox: int, oy: int, w: int, h: int):
        self._call("peer_send_atlas_rect", C.c_uint32(ox), C.c_uint32(oy), C.c_uint32(w), C.c_uint32(h))

    def peer_send_rows(self, row_begin: int, row_end: int, root: int = -1):
        self._call("peer_send_rows", C.c_uint32(row_begin), C.c_uint32(row_end), C.c_int(root))

    def peer_signal(self, kind: int):
        self._call("peer_signal", C.c_uint32(kind))

    def peer_wait(self, kind: int, expected):
        e = np.ascontiguousarray(expected, dtype=np.uint32)
        self._call("peer_wait", C.c_uint32(kind), _ptr(e))

    def set_cull_shard(self, index: int, count: int):
        self._call("set_cull_shard", C.c_uint32(index), C.c_uint32(count))

    def peer_destroy(self):
        self._call("peer_destroy")

    def clear_shadow_rect(self, ox: int, oy: int, w: int, h: int):
        self._call("clear_shadow_rect", C.c_uint32(ox), C.c_uint32(oy), C.c_uint32(w), C.c_uint32(h))

    def forward_blend(self):
        self._call("forward_blend")

    def tonemap(self, srgb_target: bool = True):
        self._call("tonemap", C.c_int(1 if srgb_target else 0))

    def set_parity_target(self, enabled: bool = True):
        self._call("set_parity_target", C.c_int(1 if enabled else 0))

    def readback_hdr_f32(self) -> np.ndarray:
        out = np.empty((self.height, self.width, 4), dtype=np.float32)
        self._call("readback_hdr_f32", _ptr(out), C.c_uint64(out.size))
        return out

    def readback_hdr_f16(self) -> np.ndarray:
        out = np.empty((self.height, self.width, 4), dtype=np.float16)
        self._call("readback_hdr_f16", _ptr(out), C.c_uint64(out.size))
        return out

    def readback_depth(self) -> np.ndarray:
        out = np.empty((self.height, self.width), dtype=np.float32)
        self._call("readback_depth", _ptr(out), C.c_uint64(out.size))
        return out

    def readback_ldr(self) -> np.ndarray:
        out = np.empty((self.height, self.width, 4), dtype=np.uint8)
        self._call("readback_ldr", _ptr(out), C.c_uint64(out.size))
        return out

    def readback_shadow_atlas(self, w: int, h: int) -> np.ndarray:
        out = np.empty((h, w), dtype=np.float32)
        self._call("readback_shadow_atlas", _ptr(out), C.c_uint64(out.size))
        return out

    def readback_hiz(self, mip: int) -> np.ndarray:
        w, h = C.c_uint32(), C.c_uint32()
        self._call("readback_hiz", C.c_uint32(mip), None, C.c_uint64(0), C.byref(w), C.byref(h))
        out = np.empty((h.value, w.value), dtype=np.float32)
        self._call("readback_hiz", C.c_uint32(mip), _ptr(out), C.c_uint64(out.size), C.byref(w), C.byref(h))
        return out

    def forward_stats(self):
        s = (C.c_uint64 * 4)()
        self._call("forward_stats", s)
        return list(s)

    def forward_light_evaluations(self) -> int:
        n = C.c_uint64()
        self._call("forward_light_evaluations", C.byref(n))
        return n.value

    def device_ptr(self, camera: int, which: int):
        p, n = C.c_void_p(), C.c_uint64()
        self._call("device_ptr", C.c_uint32(camera), C.c_int(which), C.byref(p), C.byref(n))
        return p.value or 0, n.value


def load_cuda_library() -> C.CDLL:
    """dlopen librend3_b200.so (built in-tree by __graft_entry__.build()).  No fallback."""
    if not os.path.exists(CUDA_LIB_PATH):
        raise FileNotFoundError(
            f"{CUDA_LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` first. "
            "rend3_b200 has no CPU fallback."
        )
    return C.CDLL(CUDA_LIB_PATH)


def load_cuda_backend(device: int = 0, parity_target: Optional[bool] = None) -> Backend:
    """`parity_target` switches the library's rgba32f parity instrumentation on (r3_set_parity_target); left at None it follows the
    R3_PARITY_TARGET environment variable, which only the test suite sets — bench.py and the tools run the production configuration."""
    b = Backend(load_cuda_library(), "r3_", device)
    if parity_target is None:
        parity_target = os.environ.get("R3_PARITY_TARGET", "0") not in ("", "0")
    if parity_target:
        b.set_parity_target(True)
    return b
