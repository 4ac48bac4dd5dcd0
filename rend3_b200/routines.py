"""Host-side mirror of rend3-routine's interface for the hot path, driving the C ABI.

Names, argument meaning and call order follow the reference so that the parity tests read like
rend3-test's own tests:

  GpuCuller.object_uniform_upload     rend3-routine/src/culling/culler.rs:427-529
  GpuCuller.cull (+ batch_objects)    culler.rs:531-659, 682-713; batching.rs:120-250
  ForwardRoutine / shadow rendering   forward.rs:192-315; base.rs:366-448
  FrameUniforms.new                   uniforms.rs:30-49
  BaseRenderGraph.add_to_graph        base.rs:129-185 (node order)
  TonemappingRoutine.add_to_graph     tonemapping.rs:108-147

There is no render graph here: the graph's job (ordering + resource lifetime) collapses to a
fixed, stream-ordered call sequence on one CUDA stream.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np

from . import glam
from .backend import CAMERA_VIEWPORT, CB_BAKE, CB_CULL, Backend
from .layouts import CAMERA_HEADER_DTYPE, FRAME_UNIFORMS_DTYPE, PCU_MULTISAMPLED, PCU_POSITIVE_AREA_VISIBLE
from .world import LEFT, CameraState, EvalOutput, frustum_from_matrix

f32 = np.float32


def triangle_visibility_positive(handedness: str, shadow: bool) -> bool:
    """TriangleVisibility::from_winding_and_face (culler.rs:127-149): winding = handedness.into()
    (Left -> Cw, rend3-types lib.rs:1190-1197); viewport culls Back, shadow cameras cull Front."""
    cw = handedness == LEFT
    front_culled = shadow
    # (Ccw,Back)|(Cw,Front) -> positive ; (Ccw,Front)|(Cw,Back) -> negative
    return (not cw and not front_culled) or (cw and front_culled)


def per_camera_header(camera: CameraState, camera_specifier: int, resolution: Tuple[int, int], samples: int,
                      object_count: int) -> np.ndarray:
    """PerCameraUniform header written by object_uniform_upload (culler.rs:484-505)."""
    h = np.zeros((), dtype=CAMERA_HEADER_DTYPE)
    h["view"] = camera.view.reshape(16)
    h["view_proj"] = camera.view_proj.reshape(16)
    h["shadow_index"] = camera_specifier
    h["frustum"] = camera.world_frustum
    h["resolution"] = np.array(resolution, dtype=f32)
    flags = 0
    if triangle_visibility_positive(camera.handedness, camera_specifier != CAMERA_VIEWPORT):
        flags |= PCU_POSITIVE_AREA_VISIBLE
    if samples != 1:
        flags |= PCU_MULTISAMPLED
    h["flags"] = flags
    h["object_count"] = object_count
    return h


def frame_uniforms(camera: CameraState, ambient, resolution: Tuple[int, int]) -> np.ndarray:
    """FrameUniforms::new (uniforms.rs:30-49)."""
    u = np.zeros((), dtype=FRAME_UNIFORMS_DTYPE)
    u["view"] = camera.view.reshape(16)
    u["view_proj"] = camera.view_proj.reshape(16)
    u["origin_view_proj"] = camera.origin_view_proj.reshape(16)
    u["inv_view"] = glam.inverse(camera.view).reshape(16)
    try:
        u["inv_view_proj"] = glam.inverse(camera.view_proj).reshape(16)
        u["inv_origin_view_proj"] = glam.inverse(camera.origin_view_proj).reshape(16)
    except np.linalg.LinAlgError:  # singular raw projections are never inverted on the hot path
        pass
    u["frustum"] = frustum_from_matrix(camera.proj)
    u["ambient"] = np.asarray(ambient, dtype=f32)
    u["resolution"] = np.asarray(resolution, dtype=np.uint32)
    return u


@dataclass
class BaseRenderGraphSettings:
    """base.rs:95-98."""

    ambient_color: Tuple[float, float, float, float] = (0.0, 0.0, 0.0, 0.0)
    clear_color: Tuple[float, float, float, float] = (0.0, 0.0, 0.0, 0.0)


class GpuCuller:
    """culling/culler.rs:185-714, bound to one backend context.  `max_compute_workgroups_per_dimension` stands in for
    renderer.limits (batching.rs:189): batch_objects closes a batch before it reaches that many 256-invocation workgroups."""

    def __init__(self, backend: Backend, max_compute_workgroups_per_dimension: int = 65535):
        self.backend = backend
        self.max_compute_workgroups_per_dimension = max_compute_workgroups_per_dimension

    def object_uniform_upload(self, eval_output: EvalOutput, camera: CameraState, camera_specifier: int,
                              resolution: Tuple[int, int], samples: int = 1, mode: int = CB_BAKE | CB_CULL):
        header = per_camera_header(camera, camera_specifier, resolution, samples, len(eval_output.object_buffer))
        self.backend.object_uniform_upload(camera_specifier, header, mode)

    def cull(self, eval_output: EvalOutput, camera_specifier: int):
        """add_culling_to_graph (culler.rs:682-713): batch_objects then cull."""
        self.backend.batch_objects(camera_specifier, eval_output.camera.location(), self.max_compute_workgroups_per_dimension)
        self.backend.cull(camera_specifier)


class BaseRenderGraph:
    """base.rs:103-186 collapsed to a call sequence."""

    def __init__(self, backend: Backend, max_compute_workgroups_per_dimension: int = 65535):
        self.backend = backend
        self.gpu_culler = GpuCuller(backend, max_compute_workgroups_per_dimension)
        self._resolution: Optional[Tuple[int, int]] = None

    def upload_world(self, ev: EvalOutput, device_shadow_cameras: bool = False, movable_objects: bool = False,
                     device_point_lights: bool = False):
        """What evaluate_instructions leaves in wgpu buffers (renderer/eval.rs:157-181).  With `device_shadow_cameras` the lights go up
        as sources and atlas placements; the frame evaluates their shadow cameras on the device.  With `movable_objects` the mesh
        bounding spheres go up too (r3_set_object_mesh_spheres), so that r3_set_object_transforms can move the objects.  With
        `device_point_lights` the point lights go up as PointLightManager's handle table (r3_set_point_light_sources); the frame
        evaluates them on the device."""
        b = self.backend
        b.set_objects(ev.object_buffer)
        flags = (ev.object_live & 1) | ((ev.object_atomic & 1) << 1) | ((ev.object_back_to_front & 1) << 2)
        loc = np.ascontiguousarray(ev.object_location, dtype=f32)
        b.set_object_sort_info(ev.object_material_key, flags.astype(np.uint8), loc)
        if movable_objects:
            assert ev.object_mesh_sphere is not None, "this EvalOutput carries no mesh spheres"
            b.set_object_mesh_spheres(ev.object_mesh_sphere)
        b.set_mesh_buffer(ev.mesh_buffer)
        b.set_textures(ev.texture_descs, ev.texture_texels)
        b.set_skybox(ev.skybox_desc, ev.skybox_texels)
        b.set_materials(ev.material_buffer)
        if device_shadow_cameras:
            b.set_directional_light_sources(ev.directional_sources, ev.shadow_target_size[0], ev.shadow_target_size[1], ev.camera.handedness == LEFT)
        else:
            b.set_directional_lights(ev.directional_buffer, ev.shadow_target_size[0], ev.shadow_target_size[1])
        if device_point_lights:
            b.set_point_light_sources(*ev.point_sources)
        else:
            b.set_point_lights(ev.point_buffer)

    def add_to_graph(self, ev: EvalOutput, resolution: Tuple[int, int], samples: int = 1,
                     settings: BaseRenderGraphSettings = BaseRenderGraphSettings(), srgb_target: bool = True,
                     upload: bool = True, scissor_rows: Optional[Tuple[int, int]] = None, shadow_filter=None, after_shadows=None,
                     after_target=None, tonemap: bool = True, skinning=None, frame_graph: Optional[bool] = None, before_resolve=None,
                     posed_skinning: bool = False, posed_objects: bool = False, device_shadow_cameras: bool = False, object_transforms=None,
                     movable_objects: bool = False, device_point_lights: bool = False, point_light_updates=None, object_presence=None,
                     material_updates=None, joint_matrices=None, mesh_deforms=None, remeshes=None, object_variants=None,
                     directional_changes=None, texture_writes=None):
        """One frame in the node order of base.rs:135-185.  `scissor_rows` restricts rasterisation and shading
        to a band of pixel rows (the screen-tile split of the multi-GPU forward pass); `shadow_filter(i)` selects the shadow
        maps this rank renders — it then clears only their rects, the others arrive from their owners — and `after_shadows()`
        runs once they are in the atlas (the ranks send their maps to the peers there) and `before_resolve()` right before the
        shading reads the atlas (the ranks wait for the peers' maps there: the exchange overlaps the viewport cull and raster); `after_target()` runs once the render target and
        the atlas exist (peer mappings are created there); `tonemap=False` leaves the blit to the caller (the assembling rank
        runs it after the other ranks' rows have arrived); `frame_graph` records the frame's stream work and submits it as ONE CUDA
        graph launch (r3_frame_begin / r3_frame_end; the reference submits once per frame, graph.rs:510) — default: the R3_FRAME_GRAPH
        environment variable.  `skinning` = (records, joint matrices) skins with r3_skin, which uploads the matrices and waits for the
        stream (a recorded frame flushes there); `posed_skinning` instead poses the skeletons on the device and skins from the resident
        records and joint buffer (r3_pose_skeletons + r3_skin_posed after r3_set_animations / r3_set_skeletons / r3_set_pose_jobs):
        only enqueued work, so the frame stays one graph.  `posed_objects` poses the animated nodes' objects on the device first
        (r3_pose_objects after r3_set_object_animations / r3_set_object_pose_jobs): their transforms, world spheres and sort locations
        are written before any camera culls, also enqueue only.  `device_shadow_cameras` uploads the lights as sources
        (r3_set_directional_light_sources) and evaluates their shadow cameras on the device around this frame's camera
        (r3_evaluate_shadow_cameras, r3_shadow_uniform_upload): a frame whose camera moves needs no light upload.
        `object_transforms` = (slots or None, matrices) moves objects at the skinning node, before `posed_objects`
        (Renderer::set_object_transform in bulk): CUDA tensors go through r3_set_object_transforms_device — enqueue only, their producer
        ordered on the context's stream — and host arrays through r3_set_object_transforms, which waits for the stream.  It needs the mesh
        spheres: an uploading frame with `movable_objects` (or `object_transforms`) sends them.  `device_point_lights` uploads the point
        lights as a handle table and evaluates them on the device right after the frame uniforms (r3_evaluate_point_lights, enqueue only);
        `point_light_updates` = (handles, sources, live) adds, updates and removes handles first (PointLightManager::{add, update,
        remove}): CUDA tensors through r3_update_point_light_sources_device — enqueue only, their producer ordered on the context's
        stream — and host arrays through r3_update_point_light_sources, which waits for the stream.  `object_presence` = (slots or None,
        enabled) switches prepared slots on and off at the skinning node, before `object_transforms` (ObjectManager::add into a prepared
        slot / remove): CUDA tensors through r3_set_objects_enabled_device — enqueue only — and host arrays through
        r3_set_objects_enabled, which waits for the stream.  `material_updates` = (indices or None, records) replaces materials before
        the first pass that reads them (MaterialManager::update + evaluate's scatter): CUDA tensors through r3_update_materials_device —
        enqueue only, their producer ordered on the context's stream — and host arrays through r3_update_materials, which waits for the
        stream.  A transparency change also needs the objects' sort info (r3_update_object_sort_info) before the frame.
        `joint_matrices` = (writes, mat4s, inverse_binds or None) sets skeletons' joint matrices at the skinning node
        (Renderer::set_skeleton_joint_matrices, or set_skeleton_joint_transforms with inverse binds), after the pose of `posed_skinning`
        so that an application's override (a ragdoll) wins over the clip, and then skins from the resident joint buffer (r3_skin_posed,
        after r3_set_skeletons): CUDA tensors through r3_set_joint_matrices_device — enqueue only, their producer ordered on the
        context's stream — and host arrays through r3_set_joint_matrices, which waits for the stream.
        `mesh_deforms` = positions ((n, 3) float32, every mesh of the set made by r3_set_deformable_meshes, mesh after mesh) deforms the
        set at the skinning node (the rebuild of each mesh and the re-add of its objects): before `skinning`, `object_presence`,
        `object_transforms`, `posed_objects` and the skeletons, so that a move in the same frame wins the location (set_object_transform
        after add) and a deformed skinning base is skinned from the new positions.  A CUDA tensor goes through r3_deform_meshes_device —
        enqueue only, its producer ordered on the context's stream — and a host array through r3_deform_meshes, which waits for the
        stream.
        `remeshes` = dict(counts=, positions=, indices=, and normals= / tangents= / uv0= / color0= where the set reads them) remeshes the set
        made by r3_set_remeshable_meshes (the rebuild of each mesh from new vertices and indices and the re-add of its objects) in the
        place of `mesh_deforms`; a context holds one of the two sets, so the two arguments are exclusive.  CUDA tensors go through
        r3_remesh_meshes_device (enqueue only; a mesh that fails validation is left as it was, see readback_remesh_status) and host arrays
        through r3_remesh_meshes, which waits for the stream.
        `object_variants` = (slots or None, choices) switches objects between the prepared mesh and material variants of the set made by
        r3_set_object_variants (ObjectManager::add with another mesh kind or material) at the skinning node, before `object_presence` and
        `object_transforms`: CUDA tensors through r3_switch_object_variants_device — enqueue only, their producer ordered on the
        context's stream — and host arrays through r3_switch_object_variants, which waits for the stream.
        `directional_changes` = DirectionalLightChanges (DIRECTIONAL_LIGHT_CHANGE_DTYPE records) applied to the lights of
        `device_shadow_cameras` right before their shadow cameras are evaluated (DirectionalLightManager::update): a CUDA tensor through
        r3_update_directional_light_sources_device, a host array through r3_update_directional_light_sources; both only enqueue work.
        `texture_writes` = (regions, texels) — EvalOutput.texture_writes, or TEXTURE_REGION_DTYPE rows and texel bytes a CUDA producer
        wrote — patches rectangles of the table's and the skybox's levels before the first pass that samples them (a texture added
        again each frame, in rend3): CUDA tensors through r3_write_texture_regions_device — enqueue only, their producer ordered on the
        context's stream — and host arrays through r3_write_texture_regions, which waits for the stream."""
        import os
        if frame_graph is None:
            frame_graph = os.environ.get("R3_FRAME_GRAPH", "0") not in ("", "0")
        b, culler = self.backend, self.gpu_culler
        if upload:
            self.upload_world(ev, device_shadow_cameras, movable_objects or object_transforms is not None,
                              device_point_lights or point_light_updates is not None)
        if self._resolution != (resolution, samples, tuple(settings.clear_color)):
            b.set_render_target(resolution[0], resolution[1], samples, settings.clear_color)
            self._resolution = (resolution, samples, tuple(settings.clear_color))
        if scissor_rows is not None:
            b.set_scissor_rows(scissor_rows[0], scissor_rows[1])
        if after_target is not None:
            after_target()
        if frame_graph:
            b.frame_begin()
        if shadow_filter is None:
            b.clear_shadow_atlas()                                                # base.rs:139
        else:
            for i, s in enumerate(ev.shadows):
                if shadow_filter(i):
                    b.clear_shadow_rect(s.offset[0], s.offset[1], s.size, s.size)
        b.set_frame_uniforms(frame_uniforms(ev.camera, settings.ambient_color, resolution))  # :142
        if directional_changes is not None:                                       # DirectionalLightManager::update
            assert device_shadow_cameras, "directional_changes: the lights are sources only with device_shadow_cameras"
            if getattr(directional_changes, "is_cuda", False):
                b.update_directional_light_sources_device(directional_changes)
            else:
                b.update_directional_light_sources(directional_changes)
        if device_shadow_cameras:                                                 # DirectionalLightManager::evaluate around this camera
            b.evaluate_shadow_cameras(ev.camera.location())
        if point_light_updates is not None:                                       # PointLightManager::{add, update, remove}
            handles, sources, live = point_light_updates
            if getattr(handles, "is_cuda", False):
                b.update_point_light_sources_device(handles, sources, live)
            else:
                b.update_point_light_sources(handles, sources, live)
        if device_point_lights or point_light_updates is not None:                # PointLightManager::evaluate (renderer/eval.rs:180)
            b.evaluate_point_lights()
        if mesh_deforms is not None:                                              # :145 meshes rebuilt from new positions, objects re-added
            if getattr(mesh_deforms, "is_cuda", False):
                b.deform_meshes_device(mesh_deforms)
            else:
                b.deform_meshes(mesh_deforms)
        if remeshes is not None:                                                  # :145 meshes rebuilt from new vertices and indices
            assert mesh_deforms is None, "remeshes and mesh_deforms: a context holds one dynamic-mesh set"
            if getattr(remeshes["counts"], "is_cuda", False):
                b.remesh_meshes_device(**remeshes)
            else:
                b.remesh_meshes(**remeshes)
        if skinning is not None:                                                  # :145 state.skinning: (skeleton records, joint matrices)
            b.skin(skinning[0], skinning[1])
        if texture_writes is not None:                                            # textures that change, before the shadow passes
            regions, texels = texture_writes
            if getattr(regions, "is_cuda", False):
                b.write_texture_regions_device(regions, texels)
            else:
                b.write_texture_regions(regions, texels)
        if material_updates is not None:                                          # :145 materials that change, before the shadow passes
            indices, records = material_updates
            if getattr(records, "is_cuda", False):
                b.update_materials_device(records, indices)
            else:
                b.update_materials(records, indices)
        if object_variants is not None:                                           # :145 objects re-added with another mesh or material
            slots, choices = object_variants
            if getattr(choices, "is_cuda", False):
                b.switch_object_variants_device(choices, slots)
            else:
                b.switch_object_variants(choices, slots)
        if object_presence is not None:                                           # :145 objects that appear or disappear this frame
            slots, enabled = object_presence
            if getattr(enabled, "is_cuda", False):
                b.set_objects_enabled_device(enabled, slots)
            else:
                b.set_objects_enabled(enabled, slots)
        if object_transforms is not None:                                         # :145 objects the application moved this frame
            slots, matrices = object_transforms
            if getattr(matrices, "is_cuda", False):
                b.set_object_transforms_device(matrices, slots)
            else:
                b.set_object_transforms(matrices, slots)
        if posed_objects:                                                         # :145 pose_animation_frame's set_object_transform half
            b.pose_objects()
        if posed_skinning:                                                        # :145 from resident data (r3_set_skeletons / r3_set_pose_jobs)
            b.pose_skeletons()
        if joint_matrices is not None:                                            # :145 skeletons posed by the application, over the clip
            writes, mat4s, inverse_binds = joint_matrices
            if getattr(mat4s, "is_cuda", False):
                b.set_joint_matrices_device(writes, mat4s, inverse_binds)
            else:
                b.set_joint_matrices(writes, mat4s, inverse_binds)
        if posed_skinning or joint_matrices is not None:
            b.skin_posed()
        mine = [(i, s) for i, s in enumerate(ev.shadows) if shadow_filter is None or shadow_filter(i)]
        for i, s in mine:                                                         # :148
            if device_shadow_cameras:
                b.shadow_uniform_upload(i, len(ev.object_buffer))
            else:
                culler.object_uniform_upload(ev, s.camera, i, (s.size, s.size), 1)
        for i, s in mine:                                                         # :150
            culler.cull(ev, i)
        for i, s in mine:                                                         # :153
            b.shadow_pass(i, s.offset[0], s.offset[1], s.size)
        if after_shadows is not None:
            after_shadows()
        culler.object_uniform_upload(ev, ev.camera, CAMERA_VIEWPORT, resolution, samples)   # :156
        b.forward_begin()
        b.forward_pass(0)                                                         # :159 predicted triangles
        b.hiz_build()                                                             # :162
        culler.cull(ev, CAMERA_VIEWPORT)                                          # :169
        b.forward_pass(1)                                                         # :172 residual triangles
        if before_resolve is not None:
            before_resolve()
        b.forward_resolve()                                                       # fs_main of the opaque + cutout fragments
        # skybox (:175) is outside this path
        b.forward_blend()                                                         # :181 transparent objects, back to front
        if tonemap:
            b.tonemap(srgb_target)                                                # :184
        if frame_graph:
            b.frame_end()
