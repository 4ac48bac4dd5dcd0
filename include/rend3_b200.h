/* rend3_b200.h — C ABI of librend3_b200.so: rend3's GPU-driven per-object hot path on H100.
 *
 * The library replaces, beneath rend3's public Renderer/Object/Material/RenderGraph API, the
 * work that `rend3-routine` records into wgpu for:
 *     GpuCuller::object_uniform_upload  + uniform_prep.wgsl     (culling/culler.rs:427-529)
 *     batch_objects                                              (culling/batching.rs:120-250)
 *     GpuCuller::cull                   + cull.wgsl              (culling/culler.rs:531-659)
 *     ForwardRoutine::add_forward_to_graph + opaque.wgsl/depth.wgsl (forward.rs:192-315)
 *     HiZRoutine::add_hi_z_to_graph     + hi_z.wgsl              (hi_z.rs:161-234)
 *     TonemappingRoutine::add_to_graph  + blit.wgsl              (tonemapping.rs:108-147)
 * in the node order of BaseRenderGraph::add_to_graph (base.rs:129-185).
 *
 * Conventions
 *   - every entry point returns 0 on success, a negative R3_E_* code otherwise; the message is
 *     available from r3_last_error().  Nothing unwinds, aborts or exits across the boundary
 *     (the reference panics inside graph nodes, culler.rs:439,572 — a C ABI cannot).
 *   - host pointers are borrowed for the duration of the call only; the library owns all
 *     device memory.  Buffers are the std430 bytes rend3's managers already produce
 *     (r3_layouts.h), so the Rust side uploads exactly what it uploads to wgpu today.
 *   - one context per GPU; calls on a context must be externally serialised (this is the
 *     `data_core` mutex of the reference, rend3/src/graph/graph.rs:265).  The per-frame entry points
 *     (r3_object_uniform_upload, r3_batch_objects, r3_cull, r3_shadow_pass, r3_forward_*, r3_hiz_build, r3_tonemap,
 *     r3_skin's kernel, r3_pose_skeletons, r3_skin_posed, r3_pose_objects, r3_set_object_transforms_device, r3_set_objects_enabled_device,
 *     r3_switch_object_variants_device, r3_update_materials_device, r3_set_joint_matrices_device, r3_deform_meshes_device, r3_remesh_meshes_device, r3_evaluate_shadow_cameras,
 *     r3_shadow_uniform_upload, r3_update_point_light_sources_device, r3_evaluate_point_lights, r3_update_directional_light_sources,
 *     r3_update_directional_light_sources_device, r3_write_texture_regions_device,
 *     r3_exchange_merge, r3_peer_*) only enqueue work on the
 *     context's stream and return.
 *     What BLOCKS the calling thread until the stream has drained: r3_sync, every r3_readback_*, r3_visible_count,
 *     r3_batch_counts / r3_batching_info / r3_forward_stats / r3_stage_times (small device-to-host reads), and the
 *     uploads that borrow a HOST pointer — r3_set_objects, r3_update_objects, r3_set_object_sort_info,
 *     r3_set_mesh_buffer, r3_set_materials, r3_update_materials, r3_set_textures, r3_set_skybox, r3_set_*_lights, r3_skin's joint upload,
 *     r3_set_animations, r3_set_skeletons, r3_set_pose_jobs, r3_set_joint_matrices, r3_readback_joint_matrices, r3_set_object_animations,
 *     r3_set_object_pose_jobs, r3_set_object_mesh_spheres, r3_set_object_transforms, r3_set_objects_enabled, r3_set_object_variants,
 *     r3_switch_object_variants, r3_set_deformable_meshes,
 *     r3_deform_meshes, r3_set_remeshable_meshes, r3_remesh_meshes, r3_readback_remesh_status, r3_set_directional_light_sources,
 *     r3_readback_shadow_cameras, r3_set_point_light_sources, r3_update_point_light_sources, r3_readback_point_lights,
 *     r3_write_texture_regions —
 *     because the pointer is only valid for the duration of the call (they are the counterpart of queue.write_buffer,
 *     which copies before it returns).  r3_set_objects_device borrows device memory and does not block.  A buffer that
 *     has to grow (first frame, larger world, new resolution) is reallocated with a stream synchronisation as well.
 *   - incremental world updates — r3_update_object_sort_info, r3_resize_objects, r3_update_mesh_buffer, r3_update_textures — block
 *     like the other host-pointer uploads.  Every argument is checked before anything is written: a rejected call returns
 *     R3_E_INVALID or R3_E_STATE and leaves the context as it was.  A count of 0 is a no-op.  Their result equals the full upload
 *     of the updated arrays (r3_set_object_sort_info, r3_set_objects + r3_set_object_sort_info, r3_set_mesh_buffer, r3_set_textures);
 *     what they save is the host loop and the PCIe copy of everything that did not change.  Growth keeps the old contents by a
 *     device copy, as the reference does (copy_buffer_to_buffer into the larger buffer).
 *   - `camera` is R3_CAMERA_VIEWPORT or a shadow index 0..R3_MAX_SHADOWS-1
 *     (CameraSpecifier, rend3-routine/src/common/camera.rs).
 */
#ifndef REND3_B200_H
#define REND3_B200_H

#include <stddef.h>
#include <stdint.h>

#include "r3_layouts.h"

#ifdef __cplusplus
extern "C" {
#endif

#define R3_ABI_VERSION 1u
#define R3_MAX_SHADOWS 63u

enum {
    R3_OK = 0,
    R3_E_INVALID = -1,   /* bad argument / call order (the reference's assert!/unwrap sites) */
    R3_E_CUDA = -2,      /* CUDA runtime failure; message carries cudaGetErrorString */
    R3_E_OOM = -3,       /* allocation failed (MeshCreationError::BufferAllocationFailed analogue) */
    R3_E_NO_DEVICE = -4, /* RendererInitializationError::MissingAdapter analogue */
    R3_E_STATE = -5      /* required earlier stage has not run for this camera/frame */
};

typedef struct r3_ctx r3_ctx;

/* ------------------------------------------------------------------ context */
uint32_t r3_abi_version(void);
/* replaces rend3::create_iad + GpuCuller::new/PbrRoutine::new pipeline creation (base.rs:111-124) */
int r3_ctx_create(int device, r3_ctx** out);
int r3_ctx_destroy(r3_ctx* ctx);
const char* r3_last_error(const r3_ctx* ctx);
int r3_sync(r3_ctx* ctx);
/* the CUDA stream all work of this context is enqueued on (cudaStream_t as void*) */
int r3_get_stream(r3_ctx* ctx, void** stream);
/* number of kernel launches issued by this context since creation (bench.py gpu_launches) */
int r3_launch_count(r3_ctx* ctx, uint64_t* launches);

/* Frame submission as ONE CUDA graph launch (the reference submits once per frame, rend3/src/graph/graph.rs:510).  Optional: bracket
 * the per-frame calls (r3_clear_shadow_atlas ... r3_tonemap) with r3_frame_begin / r3_frame_end.  The stream work in between is recorded
 * by stream capture instead of being launched; r3_frame_end turns it into a graph — the instantiated graph of the previous frame of the
 * same parity is updated in place (cudaGraphExecUpdate: same kernels, this frame's arguments and ping-pong pointers), so steady-state
 * frames pay no instantiation — and launches it.  A call that has to wait for the stream inside the bracket (a buffer that must grow, a
 * host-side batch_objects, a readback) submits what was recorded so far, waits, and the rest of the frame runs eagerly; results are the
 * same either way.  stats: [0] frames ended, [1] frames submitted as a graph, [2] early flushes, [3] graph (re)instantiations. */
int r3_frame_begin(r3_ctx* ctx);
int r3_frame_end(r3_ctx* ctx);
int r3_frame_graph_stats(r3_ctx* ctx, uint64_t stats[4]);

/* optional per-stage device timing (off by default): when enabled, CUDA event pairs are recorded around the kernels below and
 * r3_stage_times returns, per stage, the summed duration in ms and the number of launches since the last call (it synchronises).
 * stage ids: 0 triangle_test_kernel, 1 raster_setup_kernel (colour passes), 2 raster_setup_kernel (shadow passes), 3 raster_band_kernel,
 * 4 resolve_kernel, 5 the batch_objects sort, 6 cull_bake_kernel, 7 triangle_compact_kernel. */
int r3_set_stage_timing(r3_ctx* ctx, int enabled);
int r3_stage_times(r3_ctx* ctx, double ms[8], uint32_t launches[8]);

/* ------------------------------------------------------------------ world data
 * same bytes as the wgpu buffers named on the right */
int r3_set_objects(r3_ctx*, const r3_object* records, uint32_t n_slots);           /* object_manager.buffer::<M>() (object.rs:193) */
int r3_update_objects(r3_ctx*, const uint32_t* slots, const r3_object* records, uint32_t n); /* ScatterCopy (object.rs:344-364) */
/* borrow an object buffer that already lives in device memory (zero copy; caller keeps it alive) */
int r3_set_objects_device(r3_ctx*, const void* device_records, uint32_t n_slots);
/* facts batch_objects reads from the object/material managers (batching.rs:144-167):
 * flags bit0 = slot is live (enumerated_objects), bit1 = SortingReason::Optimization
 * ("atomic capable"), bit2 = SortingOrder::BackToFront.  location = InternalObject::location. */
int r3_set_object_sort_info(r3_ctx*, const uint64_t* material_key, const uint8_t* flags,
                            const float* location_xyz, uint32_t n_slots);
/* FreelistDerivedBuffer::apply's scatter of the stale entries (util/freelist/buffer.rs:85-97, object.rs:302-316): entry i sets slot
 * slots[i] exactly as r3_set_object_sort_info would; every slot must be below the current sort-info count.  A slot listed twice takes
 * its later entry.  Starts a new frame epoch, like the full call.  The per-frame call for objects that move (location) or change. */
int r3_update_object_sort_info(r3_ctx*, const uint32_t* slots, const uint64_t* material_key, const uint8_t* flags,
                               const float* location_xyz, uint32_t n);
/* FreelistDerivedBuffer::apply's growth (buffer.rs:66-83, object.rs:363): the object buffer grows to n_slots (never shrinks) by a device
 * copy; the new slots are zero records (enabled 0).  When sort info is set it grows too (key 0, flags 0, location 0).  Equals
 * r3_set_objects + r3_set_object_sort_info of the old contents followed by zeros.  R3_E_STATE while the records are borrowed
 * (r3_set_objects_device) or a visible-set exchange / peer plumbing is connected (their buffers are sized at creation). */
int r3_resize_objects(r3_ctx*, uint32_t n_slots);
/* Objects that move: Renderer::set_object_transform (object.rs:302-316) for n objects in one kernel, from host or device memory.
 *   r3_set_object_mesh_spheres       InternalObject::mesh_bounding_sphere (object.rs:268-270) per slot, (centre, radius): what
 *                                    set_object_transform moves to world space.  slots == NULL: spheres for slots 0 .. n-1 (replaces the
 *                                    array); otherwise entry i sets slot slots[i], each below the current sphere count and named once
 *                                    (R3_E_INVALID otherwise, nothing written).  Blocking.  The spheres belong to the mesh, not the record:
 *                                    r3_set_objects keeps them, r3_resize_objects grows them with zero spheres like the sort info.
 *   r3_set_object_transforms         transform = mat4s[i] (column-major), bounding sphere = mesh sphere.apply_transform
 *                                    (util/frustum.rs:22-32), sort location = transform_point3a(ZERO).  Arithmetic: rule R12 (DESIGN.md §2).
 *                                    slots == NULL: slots 0 .. n-1 (the dense form, n <= the slot count).  Host pointers, blocking: they are
 *                                    copied to the device, one kernel runs and the stream is drained once.
 *   r3_set_object_transforms_device  the same from DEVICE memory, enqueue only: the pointers (matrices 16-byte aligned) are read by the
 *                                    kernel when it runs on the context's stream.  Legal between r3_frame_begin and r3_frame_end; in a
 *                                    frame graph the kernel's arguments are updated in place.  Whatever produces the buffers must be
 *                                    ordered before the call on that stream (r3_get_stream: enqueue the producer there, or make the
 *                                    stream wait on an event before r3_frame_begin), and they must stay valid until the frame has run.
 * Only float4 #0-4 of the record change (transform, sphere); `enabled`, the cold fields, key and flags are untouched, exactly as in
 * r3_pose_objects.  The same kernel writes the cull + bake's dense copies of those slots (rows, row 3, spheres, the affine bit) and, when
 * sort info is set, their sort locations; a new frame epoch starts, as after a pose.  The host batching's mirror of the locations is
 * refreshed in the drain it makes anyway for the visible list; the device batching path gets no new drain.
 * Slots must be distinct (two entries' stores would land in an unspecified order).  The host form checks this, and that every slot is
 * below the current slot count, before anything is written: R3_E_INVALID, context unchanged.  The device form cannot look: out-of-range
 * slots are dropped (ScatterCopy's robust access, as in r3_update_objects), distinctness is a precondition.
 * R3_E_STATE: before r3_set_objects; while the mesh spheres cover fewer slots than the object buffer (never set, or r3_set_objects made
 * the world larger than they are); while the object buffer is borrowed (r3_set_objects_device).  n == 0 is R3_OK and enqueues nothing.
 * A slot that r3_pose_objects also poses takes whichever of the two calls is enqueued later. */
int r3_set_object_mesh_spheres(r3_ctx*, const uint32_t* slots_or_null, const float* center_radius /* n x 4 */, uint32_t n);
int r3_set_object_transforms(r3_ctx*, const uint32_t* slots_or_null, const float* mat4s /* n x 16, column-major */, uint32_t n);
int r3_set_object_transforms_device(r3_ctx*, const uint32_t* d_slots_or_null, const float* d_mat4s, uint32_t n);
/* Objects that come and go: ObjectManager::add into a slot prepared earlier, and remove (object.rs:122-160, 330-342), for n slots in one
 * kernel, from host or device memory.  The host prepares a pool once (records with mesh, material and transform, sort info with the
 * keys); each frame switches slots on and off.  Entry i makes slot slots[i] present (enabled[i] != 0) or absent (== 0): it writes the
 * record's `enabled` word (1 or 0), the slot's bit of the cull + bake's enabled bits and, when sort info is set, its live bit
 * (enumerated_objects, flags bit 0).  Nothing else changes — transform, sphere, cold fields, key, flags bits 1-2 and location stay — so
 * switching a slot on again restores it exactly.  Placing a spawned object with r3_set_object_transforms_device in the same frame is
 * independent of the order of the two calls: they write disjoint fields.
 *   slots == NULL: slots 0 .. n-1 (the dense form, n <= the slot count).
 *   r3_set_objects_enabled         host pointers, blocking.  Every slot below the slot count, none named twice, no null pointer, checked
 *                                  before anything is written (R3_E_INVALID, context unchanged).  The host's mirrors stay exact: the live
 *                                  bits of the sort flags and the count of live key-2 slots that decides whether the blend routine runs.
 *   r3_set_objects_enabled_device  the same from DEVICE memory, enqueue only; legal between r3_frame_begin and r3_frame_end (a frame graph
 *                                  updates its arguments in place).  Producer ordering as for r3_set_object_transforms_device;
 *                                  out-of-range slots are dropped, distinct slots are a precondition.  From this call until the next
 *                                  r3_set_object_sort_info the host cannot know which slots are live, so the blend routine runs whenever
 *                                  SOME slot has material key 2, present or not.  A frame without a present key-2 object then collects
 *                                  no fragments and gives the same image, but waits for the fragment count as every frame with
 *                                  transparent objects does (a recorded frame flushes there).
 * R3_E_STATE before r3_set_objects and while the object buffer is borrowed (r3_set_objects_device).  n == 0 is R3_OK and enqueues
 * nothing.  Each call starts a new frame epoch.  A later r3_update_objects, r3_set_objects or r3_update_object_sort_info of a slot
 * overwrites what these calls wrote, and the reverse.
 * Departure from the reference: rend3's remove leaves the object enumerated (live) but disabled for one frame before its handle is
 * reclaimed (handle_alloc.rs:21-29); here an absent slot is disabled and not live at once.  The image is the same (a disabled object
 * draws nothing); the batch records of that one frame differ. */
int r3_set_objects_enabled(r3_ctx*, const uint32_t* slots_or_null, const uint8_t* enabled, uint32_t n);
int r3_set_objects_enabled_device(r3_ctx*, const uint32_t* d_slots_or_null, const uint8_t* d_enabled, uint32_t n);
/* Objects that change mesh or material: re-adding an object with another mesh kind or material (ObjectManager::add, object.rs:122-160,
 * 267-284; duplicate_object with an ObjectChange, object.rs:201-218, 318) for n slots in one kernel, from host or device memory — LOD
 * chains, damage states, team or selection material swaps, impostors.  The host prepares a table of variants once (r3_object_variant:
 * mesh range, attribute offsets, material, key, flags bits 1-2, mesh sphere) and groups of consecutive variants (r3_variant_group, e.g.
 * one LOD chain); each listed slot chooses from one group, and many slots may share a group.  A switch of slot s to variant v writes what
 * re-adding the object with v's mesh and material at its current transform writes: the record's first_index, index_count,
 * material_index and attr_offset[6]; the world sphere (BoundingSphere::apply_transform of v's mesh sphere by the slot's transform, rule
 * R12) into the record and the cull + bake's copies and centre bit; the slot's mesh sphere; and, when sort info is set, key and flags bits
 * 1-2 and the sort location = the world sphere's centre (add's location).  `enabled`, the live bit, the transform, its rows and the affine
 * bit stay: a switched absent slot stays absent.
 *   r3_set_object_variants           blocking, once per set: n_variants variants, n_groups groups and n_listed (slot, group) pairs.  Records
 *                                    are not changed.  Checks everything before it writes anything; R3_E_INVALID, the context unchanged,
 *                                    for: a null pointer with a non-zero count; a variant whose index range lies outside the mesh buffer,
 *                                    whose index_count % 3 != 0, with an offset that is neither a multiple of 4 nor R3_ATTR_ABSENT, without
 *                                    a position, or with a flag bit other than 1-2; an empty group or one reaching past the variants; a slot
 *                                    at or past the slot count or named twice; a group index >= n_groups; a slot also listed by the current
 *                                    deformable or remeshable set (r3_set_deformable_meshes / r3_set_remeshable_meshes reject the reverse).
 *                                    R3_E_STATE before r3_set_objects, while the object buffer is borrowed and while
 *                                    r3_set_object_mesh_spheres does not cover every slot.  Each listed slot's invocation floor becomes the
 *                                    largest index_count of its group, so a switch to the largest level never outgrows the culling buffers
 *                                    (r3_debug_invocation_bound).  n_variants == 0 removes the set and its floors.  r3_resize_objects grows
 *                                    the per-slot arrays (new slots unlisted).
 *   r3_switch_object_variants        host pointers, blocking: one copy, one kernel, one drain.  Entry i gives slot slots[i] variant
 *                                    group.first + choices[i] of its group; slots == NULL is the dense form over slots 0 .. n-1.
 *                                    R3_E_INVALID, nothing written, for an unlisted slot, a slot named twice or choices[i] >= group.count.
 *                                    The host's mirrors of keys and flags stay exact (the blend routine and the host batching follow them).
 *   r3_switch_object_variants_device the same from DEVICE memory, enqueue only; legal between r3_frame_begin and r3_frame_end.  Producer
 *                                    ordering as for r3_set_object_transforms_device.  Unlisted slots and out-of-range choices are dropped;
 *                                    distinct slots are a precondition.  Until the next r3_set_object_sort_info or host switch the host
 *                                    cannot know the switched keys: the blend routine runs whenever some slot or some variant of the set
 *                                    has material key 2, and the device batching is only used while no variant key is >= 64.  The host
 *                                    batching reads the slots' current variants back in the drain it makes anyway and stays exact.
 *   r3_readback_object_variants      blocking: the current variant (an index into the table) of slots [first, first + n); 0xFFFFFFFF for a
 *                                    slot that is unlisted or was not switched since the set was made.
 * R3_E_STATE from both switch calls: before a set exists; after an r3_set_mesh_buffer that left the mesh buffer shorter than the set's
 * largest index end; before r3_set_objects; while the object buffer is borrowed; while r3_set_object_mesh_spheres does not cover every
 * slot.  n == 0 is R3_OK.  Each call starts a new frame epoch.  Ordering: r3_update_objects, r3_set_objects and
 * r3_update_object_sort_info of a listed slot overwrite a switch, and the reverse (the floor still bounds the slot's index_count);
 * r3_set_object_transforms* after a switch in the same frame gives the move's location with the new mesh sphere, a switch after a move
 * gives the add's location; r3_pose_objects carries its own mesh spheres, so on a slot both posed and switched the later call wins for
 * the sphere. */
int r3_set_object_variants(r3_ctx*, const r3_object_variant* variants, uint32_t n_variants, const r3_variant_group* groups, uint32_t n_groups,
                           const uint32_t* slots, const uint32_t* slot_groups, uint32_t n_listed);
int r3_switch_object_variants(r3_ctx*, const uint32_t* slots_or_null, const uint32_t* choices, uint32_t n);
int r3_switch_object_variants_device(r3_ctx*, const uint32_t* d_slots_or_null, const uint32_t* d_choices, uint32_t n);
int r3_readback_object_variants(r3_ctx*, uint32_t* out, uint32_t first, uint32_t n);
int r3_set_mesh_buffer(r3_ctx*, const void* bytes, uint64_t nbytes);               /* eval_output.mesh_buffer (mesh.rs:99) */
/* Meshes that deform every frame (cloth, flags, a water grid, soft bodies, blend shapes evaluated by a CUDA kernel), from host or device
 * memory.  rend3's meshes are immutable: the reference rebuilds such a mesh each frame (MeshBuilder::build recomputes smooth normals and
 * tangents, rend3-types/src/lib.rs:477-512, 617-837; MeshManager::add recomputes BoundingSphere::from_mesh, mesh.rs:169) and re-adds its
 * objects (ObjectManager::add, object.rs:267-284: a new world sphere, and the sort location becomes its centre).  Here the mesh stays
 * where it is and one call rewrites, for every mesh of the set, exactly what that rebuild and re-add would produce, bit for bit: the
 * positions, the normals and tangents the build computed (R3_DEFORM_NORMALS / R3_DEFORM_TANGENTS), the mesh sphere, and for every listed
 * object slot its mesh sphere, world sphere (record, cull + bake's copies and centre bit) and sort location = the world sphere's centre.
 * Transform, rows, affine bit, `enabled`, index_count, key and flags stay.  Arithmetic: rule R15 (DESIGN.md §2).  The one departure is slot
 * identity: a re-add would take a new handle and delete the old one a frame later; the image is the same.
 *   r3_set_deformable_meshes            blocking, once per set: n_meshes r3_deformable_mesh records and n_objects (slot, mesh) pairs.  It
 *                                       reads the meshes' indices back from the device, checks everything and builds each mesh's vertex
 *                                       -> corner lists on the device (a stable radix sort by vertex, in triangle order).  R3_E_INVALID, the context
 *                                       unchanged, for: a null pointer with a non-zero count; unknown flag bits; an offset that is not a
 *                                       multiple of 4; position_offset absent; R3_DEFORM_NORMALS without normal_offset; R3_DEFORM_TANGENTS
 *                                       without tangent_offset, uv0_offset or normal_offset; a range outside the mesh buffer; index_count
 *                                       not a multiple of 3; an index >= vertex_count; more than 2^31 - 1 vertices or 2^32 - 2^11 indices in
 *                                       the set; written ranges (positions, and normals / tangents when recomputed) that overlap each other
 *                                       or a read range of the set (indices, uv0 and authored normals when tangents are recomputed); an
 *                                       object mesh >= n_meshes; a slot named twice or at or past the slot count; a slot whose record does
 *                                       not draw its mesh (first_index, index_count and attr_offset[POSITION] differ); a slot listed by
 *                                       the object-variant set (r3_set_object_variants).  R3_E_STATE before
 *                                       r3_set_objects and while the object buffer is borrowed.  n_meshes == 0 removes the set.  A context
 *                                       holds one dynamic-mesh set: this call replaces a set of r3_set_remeshable_meshes, and the reverse.
 *   r3_deform_meshes                    host positions: sum(vertex_count) x 3 floats, mesh after mesh in set order (n_floats must be that
 *                                       count, R3_E_INVALID otherwise).  One copy, the kernels, one drain.
 *   r3_deform_meshes_device             the same from DEVICE memory, enqueue only; legal between r3_frame_begin and r3_frame_end (a frame
 *                                       graph updates its arguments in place).  d_positions 4-byte aligned and n_floats as above
 *                                       (R3_E_INVALID otherwise); producer ordering as for r3_set_object_transforms_device.
 *   r3_readback_deformable_mesh_spheres blocking: the mesh spheres (centre, radius) of meshes [first, first + n) from the last deform
 *                                       or remesh (zeros before it), of whichever set is current; R3_E_INVALID past the set.
 * Every call deforms every mesh of the set.  R3_E_STATE from both deform calls: before a set exists; after r3_set_mesh_buffer; after an
 * r3_update_mesh_buffer that writes into one of the set's index ranges (call r3_set_deformable_meshes again); while the object buffer is
 * borrowed (r3_set_objects_device); while r3_set_object_mesh_spheres does not cover every listed slot; while a listed slot is at or past
 * the slot count.  Both start a new frame epoch; the host batching's mirror of the locations is refreshed in the drain it makes anyway, as
 * after a move.  Ordering: r3_set_object_transforms* after a deform in the same frame gives the move's location with the new mesh sphere
 * (set_object_transform after add); r3_pose_objects takes its targets' own mesh spheres, so on a slot both posed and deformed the later
 * call wins; r3_skin / r3_skin_posed after a deform skins from the new positions. */
int r3_set_deformable_meshes(r3_ctx*, const r3_deformable_mesh* meshes, uint32_t n_meshes,
                             const uint32_t* object_slots, const uint32_t* object_meshes, uint32_t n_objects);
int r3_deform_meshes(r3_ctx*, const float* positions, uint64_t n_floats);
int r3_deform_meshes_device(r3_ctx*, const float* d_positions, uint64_t n_floats);
int r3_readback_deformable_mesh_spheres(r3_ctx*, float* out /* n x 4 */, uint32_t first, uint32_t n);
/* Meshes whose topology changes every frame (marching-cubes isosurfaces, voxel terrain chunks being dug into, fracture and cutting, holes
 * opening in cloth, GPU decimation), from host or device memory.  The reference rebuilds such a mesh each frame (MeshBuilder::build,
 * MeshManager::add) and re-adds its objects.  Here each mesh owns ranges sized by its capacities (r3_remeshable_mesh) and one call writes,
 * for every mesh of the set, what that rebuild and re-add of the new vertices and indices would produce, bit for bit under rule R15: the
 * first vertex_count entries of every attribute range, the first index_count indices, the recomputed normals and tangents and the mesh
 * sphere; for every listed slot what a deform writes (mesh sphere, world sphere, sort location) and the record's new index_count.
 * Entries past the counts stay as they were and are never drawn.  The vertex -> corner lists are rebuilt on the device by every call.
 *   r3_set_remeshable_meshes     blocking, once per set.  Checks everything before it writes anything; R3_E_INVALID, the context
 *                                unchanged, for: a null pointer with a non-zero count; the flag and offset rules of
 *                                r3_set_deformable_meshes (color0_offset included); a capacity-sized range outside the mesh buffer; written
 *                                ranges (every present attribute, and the indices) that overlap; more than 2^31 - 1 vertices or 2^32 - 2^11
 *                                indices of capacity in the set; an object mesh >= n_meshes; a slot named twice or at or past the slot
 *                                count; a listed record that does not draw its mesh (first_index, the position, normal, tangent, uv0 and
 *                                color0 offsets differ, or index_count > index_capacity); a slot listed by the object-variant set.
 *                                R3_E_STATE before r3_set_objects and while the
 *                                object buffer is borrowed.  n_meshes == 0 removes the set.  The set replaces a set of
 *                                r3_set_deformable_meshes, and the reverse; the calls of the set that is not current return R3_E_STATE.
 *                                The listed slots' index_capacity is kept as a floor of the invocation bound that sizes the culling
 *                                buffers, so a remesh back up to capacity never outgrows them.  Counts in force before the first remesh
 *                                read 0.
 *   r3_remesh_meshes             host streams: counts (n_meshes x {vertex_count, index_count}), positions (3 floats per vertex), indices,
 *                                and normals (3), tangents (3), uv0 (2) and color0 (one 4-byte word) per vertex.  Every vertex stream is
 *                                laid out at capacity strides: mesh i starts at the sum of the earlier meshes' vertex_capacity;
 *                                indices likewise by index_capacity.  n_vertices and n_indices must be the set's total capacities.  A
 *                                mesh's normals are read when it has a normal range and does not recompute them (R3_DEFORM_NORMALS
 *                                unset), tangents likewise, uv0 and color0 whenever it has those ranges; a null stream that some mesh
 *                                reads is R3_E_INVALID.  Mesh::validate (rend3-types/src/lib.rs:533-567) on every mesh: a count above
 *                                its capacity, index_count % 3 != 0 or an index >= vertex_count rejects the whole call with
 *                                R3_E_INVALID, nothing written.  One copy per stream, the kernels, one drain.
 *   r3_remesh_meshes_device      the same from DEVICE memory (4-byte aligned), enqueue only; legal between r3_frame_begin and
 *                                r3_frame_end, producer ordering as for r3_set_object_transforms_device.  The counts vary on the device
 *                                while every launch keeps its grid, so a frame graph keeps its topology.  Validation cannot return an
 *                                error here: a failing mesh and its objects are left exactly as they were (what a failed build leaves),
 *                                its status word records the first reason (R3_REMESH_*), and the other meshes are applied.
 *   r3_readback_remesh_status    blocking: status words of meshes [first, first + n) from the last remesh and, when counts_or_null is
 *                                given, the counts in force (n x {vertex_count, index_count}).  R3_E_INVALID past the set.
 * R3_E_STATE from both remesh calls: before a set exists; after r3_set_mesh_buffer; while the object buffer is borrowed; while
 * r3_set_object_mesh_spheres does not cover every listed slot; while a listed slot is at or past the slot count.  An
 * r3_update_mesh_buffer into the set's ranges invalidates nothing.  Both calls start a new frame epoch.  A later r3_update_objects of a
 * listed slot writes the host's index_count until the next remesh.  Remeshed meshes are not skinning bases: a skeleton whose ranges lie in
 * the set reads stale vertices. */
int r3_set_remeshable_meshes(r3_ctx*, const r3_remeshable_mesh* meshes, uint32_t n_meshes,
                             const uint32_t* object_slots, const uint32_t* object_meshes, uint32_t n_objects);
int r3_remesh_meshes(r3_ctx*, const uint32_t* counts, const float* positions, const uint32_t* indices, const float* normals,
                     const float* tangents, const float* uv0, const uint32_t* color0, uint64_t n_vertices, uint64_t n_indices);
int r3_remesh_meshes_device(r3_ctx*, const uint32_t* d_counts, const float* d_positions, const uint32_t* d_indices, const float* d_normals,
                            const float* d_tangents, const float* d_uv0, const uint32_t* d_color0, uint64_t n_vertices, uint64_t n_indices);
int r3_readback_remesh_status(r3_ctx*, uint32_t* status, uint32_t* counts_or_null /* n x 2 */, uint32_t first, uint32_t n);
/* Test hook: the invocation bound the culling buffers are sized with, computed now if stale: out[0] = sum over the slots of
 * round_up(max(index_count, floor) / 3, 256), out[1] = the largest term; the floor is a listed slot's index_capacity while a remeshable
 * set exists, the largest index_count of a listed slot's group while an object-variant set exists, else 0. */
int r3_debug_invocation_bound(r3_ctx*, uint64_t out[2]);
/* MeshManager::add (mesh.rs:123-184): write nbytes at byte_offset of the megabuffer (both multiples of 4).  A write past the end extends it;
 * words between the old end and byte_offset read 0.  The allocation grows to the next power of two, keeping its contents (also what
 * r3_skin wrote) — MeshManager::reallocate_buffers (mesh.rs:264-308). */
int r3_update_mesh_buffer(r3_ctx*, uint64_t byte_offset, const void* bytes, uint64_t nbytes);
int r3_set_materials(r3_ctx*, const r3_material* records, uint32_t count);         /* material_manager.archetype_view::<M>().buffer() */
/* Materials that change: MaterialManager::update and evaluate's scatter of the stale records (material.rs:163-189, 202-227), from host or
 * device memory.  Entry i replaces material indices[i] with records[i] (the 208 GpuMaterialData bytes the shading reads); indices == NULL
 * is the dense form for materials 0 .. n-1.  Nothing else changes: object records, sort info, the frame epoch and textures stay.  A
 * material's transparency key is not in its record (Material::key, pbr/material.rs:497-503): a change of transparency also needs
 * r3_update_object_sort_info of the objects that use the material, as with r3_set_materials.
 *   r3_update_materials         host pointers, blocking: one copy, one kernel, one drain.  A null pointer, an index named twice or index
 *                               0xFFFFFFFF returns R3_E_INVALID, checked before anything is written (context unchanged).  An index at or
 *                               past the table's count grows the table, as add_material does (material.rs:131-160): the records in
 *                               between are zero, the contents are kept.  The dense form with n past the count is R3_E_INVALID.  Whether
 *                               some material discards per fragment stays exact (the host keeps that one bit per material).
 *   r3_update_materials_device  the same from DEVICE memory, enqueue only; legal between r3_frame_begin and r3_frame_end (a frame graph
 *                               updates its arguments in place).  Records 16-byte aligned; producer ordering as for
 *                               r3_set_object_transforms_device.  The table cannot grow without the host: indices at or past the count are
 *                               dropped (robust access, as in r3_update_objects), the dense form with n past the count is R3_E_INVALID,
 *                               distinct indices are a precondition.  From this call until the next r3_set_materials the host cannot know
 *                               whether some material discards per fragment, so the rasteriser runs its alpha-testing kernels, which give
 *                               the same image for materials that never discard.
 * R3_E_STATE from the device form while the table is empty (before r3_set_materials or a growing host update); the host form may start a
 * table by growth.  n == 0 is R3_OK and enqueues nothing.  A later r3_set_materials replaces everything, and the reverse.  Texture slots
 * and material indices need no new check: the sampler reads 0 for a slot past the texture table, and the raster and shading kernels read
 * material 0 for an object whose material_index is past the material table.
 * r3_readback_materials copies materials [first, first + n) to the host; blocking. */
int r3_update_materials(r3_ctx*, const uint32_t* indices_or_null, const r3_material* records, uint32_t n);
int r3_update_materials_device(r3_ctx*, const uint32_t* d_indices_or_null, const r3_material* d_records, uint32_t n);
int r3_readback_materials(r3_ctx*, r3_material* out, uint32_t first, uint32_t n);
/* the bindless d2 texture table the material records index (TextureManager::add / fill, rend3/src/managers/texture.rs;
 * `textures[material.albedo_tex - 1u]`, opaque.wgsl:152-161): descriptors + one blob with every mip level.  Sampling is
 * textureSampleGrad with the linear or nearest Repeat sampler of common/samplers.rs:42-56 (trilinear, no anisotropy). */
int r3_set_textures(r3_ctx*, const r3_texture_desc* descs, uint32_t count, const void* texels, uint64_t nbytes);
/* TextureManager::add / fill (texture.rs:98-251) a range at a time: write nbytes of texels at blob_offset (16-aligned; the blob grows like the
 * mesh buffer, contents kept), then table entries [first, first + count) — first <= the current count, so a call overwrites or appends
 * but leaves no gap.  Each descriptor is checked as r3_set_textures checks it, against the blob after the write. */
int r3_update_textures(r3_ctx*, uint32_t first, const r3_texture_desc* descs, uint32_t count, uint64_t blob_offset,
                       const void* texels, uint64_t nbytes);
/* SkyboxRoutine::set_background_texture (rend3-routine/src/skybox.rs:47-60): the cube map skybox.wgsl samples wherever the depth buffer
 * still holds its clear value.  desc->width = face size (height is ignored), six faces in the order +X, -X, +Y, -Y, +Z, -Z, each with
 * its `mip_count` levels stored tightly, face after face, from desc->byte_offset.  desc == NULL removes the skybox. */
int r3_set_skybox(r3_ctx*, const r3_texture_desc* desc, const void* texels, uint64_t nbytes);
/* Textures that change (a video frame, a simulation's or a painting's output, streamed virtual-texture pages, a time-of-day sky): rend3's
 * textures are immutable (TextureManager::add, texture.rs:98-251), so there a changed texture is added again and its materials updated.
 * Here each r3_texture_region copies raw bytes, already in the target's storage format, into one rectangle of one level of a table
 * texture or a skybox face.  There is no format conversion and no mip regeneration: the other levels keep their bytes.
 *   - The element is the format's texel (R3_TEXFMT_BPP: 1, 2, 4, 8 or 16 bytes), for BC1-BC5 and BC7 a 4x4 block
 *     (R3_TEXFMT_BLOCK_BYTES), and a source row is a row of elements (a block row).  A level's bytes start after the earlier levels'
 *     R3_TEXFMT_LEVEL_BYTES; a skybox face's at sky_desc.byte_offset + f * face_bytes, the layout r3_set_skybox checks.
 *   - A region is valid when its target exists (an index below the table's count, or a face 0-5 with a skybox set), level < mip_count,
 *     width and height are above 0 and the rectangle lies inside the level; for block formats x and y are multiples of 4 and width and
 *     height multiples of 4 or reaching the level's edge (so ragged 6x6, 2x2 and 1x1 tail levels are writable); src_offset and src_pitch
 *     are multiples of the element size and src_pitch >= the row's bytes; the last source row ends within nbytes; _reserved == 0.
 *   r3_write_texture_regions         HOST pointers, blocking.  The whole call is checked first against the host's copy of the descriptors
 *                                    (which r3_set_textures and r3_update_textures keep): an invalid region, two regions of one target and
 *                                    level whose rectangles meet, or a null pointer returns R3_E_INVALID and leaves the context unchanged.
 *                                    Otherwise one copy of the regions and one of the texels go into a grow-only scratch, the two kernels
 *                                    below run and the stream is drained once (inside a frame graph that flushes, as r3_update_materials).
 *   r3_write_texture_regions_device  DEVICE pointers, enqueue only; legal between r3_frame_begin and r3_frame_end.  Regions 8-byte
 *                                    aligned; producer ordering as for r3_set_object_transforms_device.  An invalid region is dropped whole
 *                                    and the others apply.  Regions that do not overlap are a precondition: where two overlap, the bytes
 *                                    are unspecified.  Writes land in whatever blob the stream holds at that point, so they order with
 *                                    r3_set_textures / r3_update_textures by stream order.
 * Both run one planning CTA and one persistent copy grid whose sizes depend on the SM count only, so frames whose n stays above 0 keep
 * the frame graph's topology; the plan scratch grows with n and never shrinks, so only a call with a larger n than before can flush.
 * R3_E_STATE from both when there is neither a texture table nor a skybox.  n == 0 is R3_OK and launches nothing.  A later
 * r3_set_textures or r3_set_skybox replaces everything.
 * r3_readback_texels copies nbytes at byte_offset of the table's blob (skybox == 0) or the skybox's (skybox != 0, up to the end of face
 * 5) to the host; R3_E_INVALID for a range outside it.  Blocking. */
int r3_write_texture_regions(r3_ctx*, const r3_texture_region* regions, uint32_t n, const void* texels, uint64_t nbytes);
int r3_write_texture_regions_device(r3_ctx*, const r3_texture_region* d_regions, uint32_t n, const void* d_texels, uint64_t nbytes);
int r3_readback_texels(r3_ctx*, int skybox, uint64_t byte_offset, void* out, uint64_t nbytes);
int r3_set_directional_lights(r3_ctx*, const void* bytes, uint64_t nbytes,
                              uint32_t atlas_width, uint32_t atlas_height);         /* directional.rs:135-156 */
int r3_set_point_lights(r3_ctx*, const void* bytes, uint64_t nbytes);              /* point.rs:58-74 */
/* PointLightManager (rend3/src/managers/point.rs) on the device: the handle table `data: Vec<Option<PointLight>>` lives in device memory
 * and its evaluate (point.rs:58-74, called once per frame at renderer/eval.rs:180) runs as a kernel, so lights that move every frame —
 * also lights whose positions a CUDA producer computes — need no upload and no stream drain.
 *   r3_set_point_light_sources            blocking: replaces the whole table with n_handles entries (data after a run of add's);
 *                                         live_or_null[h] == 0 marks handle h dead (None), live_or_null == NULL: every handle is live.
 *   r3_update_point_light_sources         blocking: add / update / remove of n handles from HOST memory.  live[i] == 0 removes handles[i],
 *                                         any other value adds or replaces it with lights[i].  A handle at or beyond the table's size grows
 *                                         the table (add's resize); the handles between start dead.  A handle named twice, a null pointer
 *                                         or the handle 0xFFFFFFFF (the table size would not fit 32 bits) is R3_E_INVALID and nothing is
 *                                         written.  The arrays are copied, one kernel runs and the stream is drained once.
 *   r3_update_point_light_sources_device  the same from DEVICE memory, enqueue only (legal between r3_frame_begin and r3_frame_end; in a
 *                                         frame graph the kernel's arguments are updated in place).  d_live_or_null == NULL: every listed
 *                                         handle is added or replaced.  Handles must be distinct (two entries' stores would land in an
 *                                         unspecified order); handles at or beyond the table's size are dropped (the table cannot grow
 *                                         without the host).  The producer of the arrays is ordered as for r3_set_object_transforms_device.
 *   r3_evaluate_point_lights              enqueue only: ShaderPointLightBuffer (count @0, then {position.xyz 1, colour * intensity, radius}
 *                                         per live handle in ascending handle order @16) into the buffer the shading reads.  Call it once
 *                                         per frame after r3_set_frame_uniforms.  Arithmetic: DESIGN.md §2, R14 (exact).
 *   r3_readback_point_lights              blocking: the buffer the shading reads, in the layout above, whichever call filled it: the first
 *                                         min(capacity_bytes, 16 + 32 count) bytes (capacity_bytes >= 16; read the count at @0 and call
 *                                         again with more room when the array did not fit).
 * r3_set_point_lights and the source calls each replace what the other set: r3_set_point_lights empties the handle table, and an
 * evaluation rewrites the buffer from the table.  After a set or update, r3_forward_resolve and r3_forward_blend return R3_E_STATE until
 * r3_evaluate_point_lights has run.  The shading reads the light count from the device buffer; the host only knows a capacity (the
 * table size, or r3_set_point_lights' count), so a frame graph keeps its topology while lights come and go. */
int r3_set_point_light_sources(r3_ctx*, const r3_point_light_source* lights, const uint8_t* live_or_null, uint32_t n_handles);
int r3_update_point_light_sources(r3_ctx*, const uint32_t* handles, const r3_point_light_source* lights, const uint8_t* live, uint32_t n);
int r3_update_point_light_sources_device(r3_ctx*, const uint32_t* d_handles, const r3_point_light_source* d_lights,
                                         const uint8_t* d_live_or_null, uint32_t n);
int r3_evaluate_point_lights(r3_ctx*);
int r3_readback_point_lights(r3_ctx*, void* bytes, uint64_t capacity_bytes);
/* DirectionalLightManager::evaluate (directional.rs:99-157) on the device, with the shadow camera arithmetic of rule R13 (DESIGN.md §2).
 *   r3_set_directional_light_sources  blocking: the lights and their atlas placements.  Fills the light buffer's static fields
 *                                     (colour * intensity, direction, 1 / atlas size, offset / atlas size, size / atlas size) and
 *                                     allocates the atlas as r3_set_directional_lights does.  Checked first: n <= R3_MAX_SHADOWS, every
 *                                     size > 0 and every placement inside the atlas; a rejected call (R3_E_INVALID) leaves the context as
 *                                     it was.  This call and r3_set_directional_lights each replace what the other set.
 *   r3_evaluate_shadow_cameras        enqueue only: one kernel writes every light's view_proj into the light buffer and its shadow camera
 *                                     (view, view_proj, frustum) into a device-resident block, around viewport_location.  Call it once
 *                                     per frame after r3_set_frame_uniforms; in a frame graph the kernel's arguments are updated in place.
 *   r3_shadow_uniform_upload          enqueue only: r3_object_uniform_upload for camera shadow_index, with view, view_proj and frustum
 *                                     read on the device from that block.  resolution = (size, size), flags from the handedness
 *                                     (single-sampled; shadow cameras cull front faces).  R3_E_STATE before sources are set or before an
 *                                     evaluation since they were set; R3_E_INVALID for shadow_index >= n or object_count > the slots.
 *   r3_readback_shadow_cameras        blocking: the first n evaluated headers (object_count 0: it is given per upload) and, unless null,
 *                                     the light records. */
int r3_set_directional_light_sources(r3_ctx*, const r3_directional_light_source* lights, uint32_t n, uint32_t atlas_width,
                                     uint32_t atlas_height, uint32_t left_handed);
int r3_evaluate_shadow_cameras(r3_ctx*, const float viewport_location[3]);
int r3_shadow_uniform_upload(r3_ctx*, uint32_t shadow_index, uint32_t object_count, uint32_t mode);
int r3_readback_shadow_cameras(r3_ctx*, r3_camera_header* out, r3_directional_light* lights_or_null, uint32_t n);
/* DirectionalLightManager::update (directional.rs:91-93, Renderer::update_directional_light at renderer/mod.rs:369) on the lights of the
 * current set: entry i applies the fields of changes[i].mask to the light at shadow index changes[i].index, as update_from_changes does.
 * Entries apply in array order and a later entry's fields override an earlier one's, as consecutive update_directional_light calls queued
 * in one frame do, so an index named twice is legal.  An empty mask changes nothing.  Nothing is clamped: NaN, inf, a negative intensity,
 * a zero direction, a direction along +-Y and distance 0 reach R13 as given, with its degenerate results.  One kernel (one thread per
 * light) rewrites the sources and the light records' colour * intensity (the single multiply of r3_set_directional_light_sources) and
 * direction; view_proj and the shadow cameras come from the next r3_evaluate_shadow_cameras, which reads distance and direction.
 *   r3_update_directional_light_sources         HOST memory, enqueue only: legal between r3_frame_begin and r3_frame_end.  Checked first:
 *                                               a non-null pointer when n > 0, every index < the light count, no mask bit outside
 *                                               R3_DIR_CHANGE_*; a rejected call returns R3_E_INVALID and enqueues nothing.  The entries
 *                                               travel as kernel parameters, 64 per launch (n > 64: consecutive launches in array order);
 *                                               nothing is copied to the device and nothing waits, so `changes` is free on return.
 *                                               Frames whose n stays within 1 .. 64 launch one kernel each and keep the frame graph's
 *                                               topology, so the graph is updated in place.  The host copy of the sources follows.
 *   r3_update_directional_light_sources_device  DEVICE memory (4-byte aligned), enqueue only; producer ordering as for
 *                                               r3_set_object_transforms_device.  An entry whose index is at or past the light count, or
 *                                               whose mask has an unknown bit, is dropped whole.  The host copy of colour, intensity,
 *                                               direction and distance is stale afterwards; the host reads only each light's `size`
 *                                               (r3_shadow_uniform_upload), which neither form changes.
 * R3_E_STATE from both unless the lights came from r3_set_directional_light_sources (none yet, or r3_set_directional_lights since).
 * n == 0 is R3_OK and launches nothing.  After an update, r3_shadow_uniform_upload, r3_readback_shadow_cameras, r3_forward_resolve and
 * r3_forward_blend return R3_E_STATE until r3_evaluate_shadow_cameras has run.  A later r3_set_directional_light_sources replaces
 * everything.  Resolution is not a field here: a new resolution, like an added or removed light, re-packs the atlas (shadow_alloc.rs), so
 * it goes through r3_set_directional_light_sources with the new placements. */
int r3_update_directional_light_sources(r3_ctx*, const r3_directional_light_change* changes, uint32_t n);
int r3_update_directional_light_sources_device(r3_ctx*, const r3_directional_light_change* d_changes, uint32_t n);
int r3_set_frame_uniforms(r3_ctx*, const r3_frame_uniforms* uniforms);             /* uniforms.rs:94-106 */

/* ------------------------------------------------------------------ GPU skinning
 * add_skinning_to_graph / GpuSkinner::execute_pass (rend3-routine/src/skinning.rs:54-199) + skinning.wgsl:37-94:
 * 4-joint linear blend of position / normal / tangent from the unskinned attribute ranges into the skeleton's
 * overridden ranges of the mesh buffer, one launch for all skeletons.  joint_matrices = global_joint_count mat4. */
int r3_skin(r3_ctx*, const r3_skinning_input* inputs, uint32_t n_skeletons, const float* joint_matrices, uint32_t n_joints);
int r3_readback_mesh_buffer(r3_ctx*, void* bytes, uint64_t capacity_bytes);

/* ------------------------------------------------------------------ skeletal animation on the device
 * The joint half of rend3-anim's pose_animation_frame (rend3-anim/src/lib.rs:165-176, 190, 214-262) with the arithmetic of rule R12
 * (DESIGN.md §2), and skinning from joint matrices that stay in device memory.  The object-transform half (lib.rs:192-212) is the next
 * block (r3_pose_objects).
 *   r3_set_animations  the skins, their joints, the clips and their key channels (blocking upload).
 *   r3_set_skeletons   r3_skin's arguments, kept resident: the skinning records and the joint buffer, which starts with the given
 *                      matrices (Skeleton::joint_matrices at creation).  Blocking.
 *   r3_set_pose_jobs   which skin is posed with which clip at which time, and which skeleton ranges receive it.  Blocking; call it
 *                      before r3_frame_begin like the other world uploads.  r3_set_animations / r3_set_skeletons drop the jobs.
 *   r3_pose_skeletons  enqueue only: every job's joint matrices into the joint buffer; ranges no job targets keep their matrices.
 *   r3_skin_posed      enqueue only: r3_skin's kernel over the resident records and joint buffer.
 * Validation: every argument is checked before anything is written; a rejected call returns R3_E_INVALID (R3_E_STATE when the data it
 * depends on is not set) and leaves the context as it was.  The reference's panics are errors: an empty key channel, fewer values than
 * key times, a NaN or negative clip duration, a target joint count above the skin's, a target outside the joint buffer, a clip / skin /
 * joint / channel / key index out of range, an order that is not a permutation listing parents first.  Departures: key times must be
 * finite, >= 0 and strictly increasing (glTF requires it), so that a binary search finds the reference's "first key with time > t";
 * the targets of all jobs (those with joint_count > 0) must write disjoint joint ranges, since the order in which two jobs' stores
 * land is unspecified.  Skins may share joint records (their ranges may overlap); each skin's topological order is its own stretch
 * of `order`, read from first_joint, and must be a parents-first permutation of that skin's joints. */
typedef struct r3_anim_library {
    const r3_anim_skin* skins; uint32_t n_skins;
    const r3_anim_joint* joints; uint32_t n_joints;
    const uint32_t* order;        /* n_joints: per skin, its joint indices in topological order (see r3_anim_skin) */
    const r3_anim_clip* clips; uint32_t n_clips;
    const r3_anim_channel* channels; uint32_t n_channels;
    const float* keys; uint64_t n_keys;   /* key times and values of every track */
} r3_anim_library;
int r3_set_animations(r3_ctx*, const r3_anim_library* library);
int r3_set_skeletons(r3_ctx*, const r3_skinning_input* inputs, uint32_t n_skeletons, const float* joint_matrices, uint32_t n_joints);
int r3_set_pose_jobs(r3_ctx*, const r3_pose_job* jobs, uint32_t n_jobs, const r3_pose_target* targets, uint32_t n_targets);
int r3_pose_skeletons(r3_ctx*);
int r3_skin_posed(r3_ctx*);
int r3_readback_joint_matrices(r3_ctx*, float* out /* n x 16 */, uint32_t first, uint32_t n);
/* Skeletons posed by the application (IK, ragdolls, blended clips, crowd simulations): Renderer::set_skeleton_joint_matrices /
 * set_skeleton_joint_transforms (rend3/src/renderer/mod.rs:302-337, managers/skeleton.rs:151-162) for many skeletons in one kernel, from
 * host or device memory, into the resident joint buffer that r3_skin_posed reads.  Write i (r3_joint_write) fills joints
 * [joint_matrix_base_offset, + joint_count) of the buffer:
 *   inverse_binds == NULL  set_skeleton_joint_matrices: mat4s[first_matrix + k] copied bit for bit (NaN payloads and -0.0 survive);
 *   otherwise              set_skeleton_joint_transforms (Skeleton::compute_joint_matrices, rend3-types/src/lib.rs:1233-1239):
 *                          mat4s[first_matrix + k] * inverse_binds[first_inverse_bind + k], rule R12's Mat4 x Mat4 (DESIGN.md §2), the
 *                          product r3_pose_skeletons stores, bit for bit.
 * Matrices are column-major, 16 floats each.  Several writes may read one source range.  A write with joint_count == 0 does nothing
 * (its offsets are not checked);
 * ranges no write names keep their matrices; nothing but the joint buffer changes.  On any range the later of this call and
 * r3_pose_skeletons wins (a ragdoll overriding the clip is written after the pose); r3_set_skeletons replaces the whole buffer.
 *   r3_set_joint_matrices         host pointers, blocking: one copy, one kernel, one drain.  R3_E_INVALID, nothing written, for a null
 *                                 pointer whose count is not 0 (writes, mat4s, inverse binds), a destination outside the joint buffer, a
 *                                 source outside n_mat4s or n_inverse_binds, two writes whose destinations overlap.
 *   r3_set_joint_matrices_device  the same from DEVICE memory, enqueue only; legal between r3_frame_begin and r3_frame_end (a frame graph
 *                                 updates its arguments in place).  The counts come from the host; a write whose destination or sources
 *                                 fall outside them or the joint buffer is dropped whole (robust access, as in the other _device calls);
 *                                 distinct destinations are a precondition.  mat4s and inverse binds 16-byte aligned, writes 4-byte
 *                                 aligned (R3_E_INVALID otherwise); producer ordering as for r3_set_object_transforms_device.
 * R3_E_STATE before r3_set_skeletons.  n_writes == 0 is R3_OK and enqueues nothing. */
int r3_set_joint_matrices(r3_ctx*, const r3_joint_write* writes, uint32_t n_writes, const float* mat4s, uint32_t n_mat4s,
                          const float* inverse_binds_or_null, uint32_t n_inverse_binds);
int r3_set_joint_matrices_device(r3_ctx*, const r3_joint_write* d_writes, uint32_t n_writes, const float* d_mat4s, uint32_t n_mat4s,
                                 const float* d_inverse_binds_or_null, uint32_t n_inverse_binds);

/* ------------------------------------------------------------------ object animation on the device
 * The object-transform half of rend3-anim's pose_animation_frame (rend3-anim/src/lib.rs:181-212): every posed node's TRS matrix becomes
 * its objects' transform, as Renderer::set_object_transform sets it (object.rs:302-316): transform, world bounding sphere
 * (mesh_bounding_sphere.apply_transform, util/frustum.rs:22-32) and sort location (transform_point3a(ZERO)).  Arithmetic: rule R12
 * (DESIGN.md §2).  Independent of the skeletal block: each set_* call drops only its own jobs.
 *   r3_set_object_animations  the nodes' bind poses, the clips, their channels and keys, and the renderer's handedness (blocking).
 *   r3_set_object_pose_jobs   r3_pose_job records (clip, time, targets) over r3_object_pose_target records.  Blocking; call it before
 *                             r3_frame_begin.  Its buffers only grow.
 *   r3_pose_objects           enqueue only: each target's record (transform and sphere, float4 #0-4; enabled and the cold fields are
 *                             untouched) and, when sort info is set, its sort location; then the cull + bake's dense copies of those
 *                             slots and a new frame epoch.  Targets whose slot is at or past the current slot count are skipped.
 *   r3_readback_objects       blocking: records [first, first + n) and, unless null, their sort locations (3 floats each).
 * Validation (include/r3_anim_check.h): R3_E_INVALID for an index out of range, a NaN or negative duration, a track as
 * r3_set_animations checks it, a target channel >= its clip's channel_count, a slot >= the current slot count, one slot named by two
 * targets of the jobs (their stores would land in an unspecified order); R3_E_STATE for jobs before the library, r3_pose_objects before
 * r3_set_objects or before the jobs, and any of these calls while the object buffer is borrowed (r3_set_objects_device).  A rejected
 * call leaves the context as it was.
 * A later r3_update_objects / r3_update_object_sort_info of a posed slot writes the bytes it is given over the pose until the next
 * r3_pose_objects, which runs at the skinning node of every frame, before any camera culls (INTEGRATION.md). */
typedef struct r3_anim_object_library {
    const r3_anim_node* nodes; uint32_t n_nodes;
    const r3_anim_node_clip* clips; uint32_t n_clips;
    const r3_anim_node_channel* channels; uint32_t n_channels;
    const float* keys; uint64_t n_keys;   /* key times and values of every track */
    uint32_t left_handed;                 /* renderer.handedness == Handedness::Left: scale.z = -scale.z (lib.rs:201-203) */
} r3_anim_object_library;
int r3_set_object_animations(r3_ctx*, const r3_anim_object_library* library);
int r3_set_object_pose_jobs(r3_ctx*, const r3_pose_job* jobs, uint32_t n_jobs, const r3_object_pose_target* targets, uint32_t n_targets);
int r3_pose_objects(r3_ctx*);
int r3_readback_objects(r3_ctx*, r3_object* out, float* locations_or_null /* n x 3 */, uint32_t first, uint32_t n);

/* ------------------------------------------------------------------ per-object cull + uniform bake
 * GpuCuller::object_uniform_upload (culler.rs:427-529) fused with the sphere-frustum test of
 * batch_objects (batching.rs:144-148, util/frustum.rs:148-161): for every slot < object_count
 * bakes MV/MVP when `enabled`, and appends the slot to the camera's ascending visible list when
 * it is live and its world sphere is inside the 5 planes. */
#define R3_CB_BAKE 1u
#define R3_CB_CULL 2u
int r3_object_uniform_upload(r3_ctx*, uint32_t camera, const r3_camera_header* header, uint32_t mode);
int r3_visible_count(r3_ctx*, uint32_t camera, uint32_t* count);
int r3_readback_visible(r3_ctx*, uint32_t camera, uint32_t* out, uint32_t capacity, uint32_t* count);
int r3_readback_object_matrices(r3_ctx*, uint32_t camera, r3_object_matrices* out, uint32_t first, uint32_t n);

/* ------------------------------------------------------------------ batching + per-triangle cull
 * batch_objects (batching.rs:120-250) over the camera's visible list: sort by ShaderJobSortingKey,
 * pack <=256 objects per ShaderBatchData, split regions on key change, remember each object's
 * global invocation for next frame.  `viewport_location` = viewport_camera_state.location(). */
int r3_batch_objects(r3_ctx*, uint32_t camera, const float viewport_location[3], uint32_t max_dispatch_count);
int r3_batch_counts(r3_ctx*, uint32_t camera, uint32_t* n_batches, uint32_t* n_regions, uint32_t* total_invocations);
int r3_readback_batches(r3_ctx*, uint32_t camera, r3_batch_data* batches, r3_region* regions);
/* which implementation of batch_objects ran last for this camera, and what it built: info[0] = 0 none / 1 on the device (radix sort +
 * block scans, no host sync; batches split at the max_dispatch_count x 256 limit of batching.rs:196 as on the host) / 2 on the host
 * (material keys >= 64, >= 2^24 slots, or R3_HOST_BATCHING set) / 3 on the device, order taken from the
 * frame-wide sort the cameras of one frame share (the sort key does not depend on the camera, batching.rs:156-157); info[1] = device overflow flag (always 0:
 * the batch tables are sized by a proven bound; kept as a tripwire); info[2] = batches, info[3] = regions.  Blocks (one 32-byte readback). */
int r3_batching_info(r3_ctx*, uint32_t camera, uint32_t info[4]);
/* GpuCuller::cull (culler.rs:531-659) + cull.wgsl.  batches/regions == NULL uses the jobs of the last
 * r3_batch_objects call; otherwise the caller's own ShaderBatchDatas (a Rust batch_objects). */
int r3_cull(r3_ctx*, uint32_t camera, const r3_batch_data* batches, uint32_t n_batches,
            const r3_region* regions, uint32_t n_regions);
/* CullingBuffers readback (culler.rs:88-125).  `partition`: 0 = Output (predicted, kept for next
 * frame), 1 = Input (residual / previous frame).  Sizes in elements. */
int r3_readback_indices(r3_ctx*, uint32_t camera, int partition, uint32_t* out, uint64_t capacity, uint64_t* count);
int r3_readback_draw_calls(r3_ctx*, uint32_t camera, int partition, r3_indirect_call* out, uint32_t capacity, uint32_t* count);
int r3_readback_culling_results(r3_ctx*, uint32_t camera, int partition, uint32_t* out, uint64_t capacity, uint64_t* count);

/* ------------------------------------------------------------------ forward path
 * render targets of BaseRenderGraphIntermediateState::new (base.rs:212-290): hdr colour rgba16f,
 * depth32f (reverse-Z, cleared to 0.0, compare GreaterEqual), shadow atlas depth32f. */
int r3_set_render_target(r3_ctx*, uint32_t width, uint32_t height, uint32_t samples, const float clear_color[4]);
int r3_clear_shadow_atlas(r3_ctx*);                                                /* clear.rs / base.rs:293-295 */
/* pbr_shadow_rendering (base.rs:366-396): depth.wgsl over the shadow camera's culled list, into
 * the atlas viewport (offset, size). */
int r3_shadow_pass(r3_ctx*, uint32_t shadow_index, uint32_t offset_x, uint32_t offset_y, uint32_t size);
/* begin the primary render pass: colour = clear colour, depth = 0.0 (base.rs:257-264) */
int r3_forward_begin(r3_ctx*);
/* ForwardRoutine::add_forward_to_graph for the opaque + cutout routines.
 * source 0 = CullingSource::Predicted (last frame's list, forward.rs:224-232),
 *        1 = CullingSource::Residual (this frame's residual list, forward.rs:212-222). */
int r3_forward_pass(r3_ctx*, int source);
int r3_hiz_build(r3_ctx*);                                                          /* hi_z.rs:161-234 */
/* run opaque.wgsl::fs_main for the winning fragment of every covered pixel */
int r3_forward_resolve(r3_ctx*);
/* pbr_forward_rendering_transparent (base.rs:181,450-466): the blend routine (pbr/routine.rs:129; material key 2,
 * BlendState::ALPHA_BLENDING, depth test + write) over this frame's residual list, whose non-atomic regions keep the
 * back-to-front object order of batch_objects (cull.wgsl:374-380).  Call after r3_forward_resolve: it blends into the
 * shaded rgba16f target.  A no-op when no object carries material key 2. */
int r3_forward_blend(r3_ctx*);
int r3_tonemap(r3_ctx*, int srgb_target);                                           /* tonemapping.rs:108-147 */

/* Parity instrumentation, OFF by default: when enabled the shading kernels also store their f32 result before the rgba16f rounding
 * (16 B per pixel more than the reference's targets write) so that tests can hold fs_main to 1e-4 without the half-precision step.
 * r3_readback_hdr_f32 fails with R3_E_STATE while it is off. */
int r3_set_parity_target(r3_ctx*, int enabled);
int r3_readback_hdr_f32(r3_ctx*, float* rgba, uint64_t capacity_floats);            /* pre-f16 shading result (parity target) */
int r3_readback_hdr_f16(r3_ctx*, uint16_t* rgba, uint64_t capacity_halfs);          /* the Rgba16Float target */
int r3_readback_depth(r3_ctx*, float* depth, uint64_t capacity);
int r3_readback_ldr(r3_ctx*, uint8_t* rgba8, uint64_t capacity);
int r3_readback_shadow_atlas(r3_ctx*, float* depth, uint64_t capacity);
int r3_readback_hiz(r3_ctx*, uint32_t mip, float* depth, uint64_t capacity, uint32_t* width, uint32_t* height);
/* forward statistics of the last frame: [0] triangles set up, [1] fragments rasterised (covered samples sent
 * to the depth test), [2] fragments shaded by r3_forward_resolve (fs_main invocations), [3] sample fragments blended by
 * r3_forward_blend (depth-test survivors of the blend routine) */
int r3_forward_stats(r3_ctx*, uint64_t stats[4]);
/* surface_shading evaluations (opaque.wgsl:440-468) of the last r3_forward_resolve, summed over its fragments (single-sampled targets):
 * directional lights + the point lights that survived the tile culling and the per-fragment range test — the flop count of the pass */
int r3_forward_light_evaluations(r3_ctx*, uint64_t* evaluations);

/* ------------------------------------------------------------------ multi-GPU plumbing
 * raw device views so torch.distributed / NCCL can move the visible list and tile rows without a
 * host bounce.  which: 0 visible list (u32), 1 hdr f16 colour, 2 object matrices, 3 visible count (u32),
 * 4 visibility words (1 bit per object slot, bit i of word w = slot 32*w + i), 5 shadow atlas (depth32f: ranks that render
 * different shadow maps merge them with an integer MAX all-reduce, the atlas being cleared to 0.0) */
int r3_device_ptr(r3_ctx*, uint32_t camera, int which, void** device_ptr, uint64_t* nbytes);
/* Exchange of the visible set between the GPUs of one node over NVLink / NVSwitch peer memory (one process per GPU, objects
 * sharded in contiguous ranges, SURVEY 8e).  r3_exchange_create allocates this rank's buffer — epoch flags, acknowledgements and
 * rows[4][n_ranks][words_per_rank] (1 bit per object slot, rows 256-byte aligned, four row sets) — and returns its CUDA IPC handle; the
 * caller all-gathers the handles with whatever it already uses (torch.distributed, MPI) and hands them to r3_exchange_connect.  From then on
 * every r3_object_uniform_upload(CULL) on that camera is one EPOCH e: its compaction kernel also stores the visibility words into row
 * (e % 4, my_rank) of EVERY rank's buffer and publishes them with flags[e % 4][my_rank] = e (st.release.sys, after system-scope fences) —
 * no collective kernel runs.  Consumers run on the context's least-priority side stream, chained on the flags ON THE DEVICE (ld.acquire.sys,
 * no host barrier), overlapping the next culls: r3_exchange_count (visible objects of every shard) and r3_exchange_merge (the global
 * ascending visible list; r3_exchange_merged hands out its device pointers, rank_base == NULL numbers the shards r * max_objects_per_rank).
 * A consumer acknowledges its epoch to every producer; a producer that is about to overwrite a row set waits — on the device — until the
 * epoch it held has been acknowledged by all ranks.  Protocol: the ranks cull in lockstep and an epoch that one rank consumes, every rank
 * consumes (the acknowledgements are awaited on that assumption); consumers may lag up to three epochs before a producer blocks. */
#define R3_IPC_HANDLE_BYTES 64
int r3_exchange_create(r3_ctx*, uint32_t camera, uint32_t n_ranks, uint32_t my_rank, uint32_t max_objects_per_rank,
                       uint8_t handle_out[R3_IPC_HANDLE_BYTES]);
int r3_exchange_connect(r3_ctx*, uint32_t camera, const uint8_t* handles /* n_ranks x R3_IPC_HANDLE_BYTES, rank order */);
/* rows [n_ranks][words_per_rank] of the LAST epoch in this rank's buffer (complete for a host reader after a stream sync + a barrier) */
int r3_exchange_words(r3_ctx*, uint32_t camera, void** device_ptr, uint64_t* nbytes, uint32_t* words_per_rank);
int r3_exchange_merge(r3_ctx*, uint32_t camera, const uint32_t* rank_objects /* n_ranks */, const uint32_t* rank_base /* n_ranks or NULL */);
int r3_exchange_merged(r3_ctx*, uint32_t camera, void** device_list /* u32 global ids */, void** device_count /* u32 */, uint64_t* capacity);
/* the light consumer: waits for the flags like r3_exchange_merge but only counts — visible objects of every shard and their total — without
 * expanding the list (4 B per visible object of the WHOLE world on every rank: a cost that grows with the number of ranks);
 * r3_exchange_counts reads counts[0 .. n_ranks] (the last one is the total) back, blocking */
int r3_exchange_count(r3_ctx*, uint32_t camera, const uint32_t* rank_objects /* n_ranks */);
int r3_exchange_counts(r3_ctx*, uint32_t camera, uint32_t* counts /* n_ranks + 1 */);
int r3_exchange_destroy(r3_ctx*, uint32_t camera);
/* Peer-memory plumbing of the multi-GPU forward pass (SURVEY 8e: shadow maps split by light, screen split in row tiles; one process per
 * GPU on one NVLink / NVSwitch node).  r3_peer_create (after r3_set_directional_lights and r3_set_render_target: the atlas and the rgba16f
 * target must exist and must not be reallocated afterwards; the objects must be uploaded) returns four CUDA IPC handles — flag block,
 * shadow atlas, colour target, staging arrays of the sharded triangle test; the
 * caller all-gathers them and calls r3_peer_connect.  Then, all stream-ordered and without host synchronisation:
 *   r3_peer_send_atlas_rect  copies a rect of the local atlas into the same rect of EVERY peer's atlas (plain stores over NVLink);
 *   r3_peer_send_rows        copies rows of the local rgba16f target into the peers' targets (root >= 0: only into that rank's);
 *   r3_peer_signal(kind)     publishes everything sent so far: flags[kind][my_rank] = ++epoch on every rank (st.release.sys);
 *   r3_peer_wait(kind, e[])  a one-CTA kernel on this context's stream that spins (ld.acquire.sys) until flags[kind][r] >= e[r] for all r.
 * kinds: 0 shadow atlas, 1 colour rows, 2 frame done, 3 visibility words of the sharded triangle test (used by r3_cull itself).  rend3_b200/parallel.py::ForwardSplit shows the per-frame protocol. */
int r3_peer_create(r3_ctx*, uint32_t n_ranks, uint32_t my_rank, uint8_t handles_out[4 * R3_IPC_HANDLE_BYTES]);
int r3_peer_connect(r3_ctx*, const uint8_t* handles /* n_ranks x 4 x R3_IPC_HANDLE_BYTES, rank order */);
/* SURVEY 8e "triangle cull: shard by batch": with count = n_ranks (> 1), r3_cull of the VIEWPORT camera tests only this rank's run of
 * workgroups — they are laid out batch after batch, so a shard is a run of batches — stores its visibility words into the staging arrays
 * of every rank, publishes them (flag kind 3) and, once everybody's words have arrived, continues with the scan / compaction on the full
 * set: every rank ends up with the same index lists and draw records.  Falls back to testing everything while translucent (non-atomic)
 * objects exist, whose in-place index slots are not exchanged. */
int r3_set_cull_shard(r3_ctx*, uint32_t shard_index, uint32_t shard_count);
int r3_peer_send_atlas_rect(r3_ctx*, uint32_t offset_x, uint32_t offset_y, uint32_t width, uint32_t height);
int r3_peer_send_rows(r3_ctx*, uint32_t row_begin, uint32_t row_end, int root /* -1 = every peer */);
int r3_peer_signal(r3_ctx*, uint32_t kind);
int r3_peer_wait(r3_ctx*, uint32_t kind, const uint32_t* expected_epochs /* n_ranks */);
int r3_peer_destroy(r3_ctx*);
/* clear one shadow map's rect (a rank that renders only some of the lights clears only theirs; the others arrive from their owners) */
int r3_clear_shadow_rect(r3_ctx*, uint32_t offset_x, uint32_t offset_y, uint32_t width, uint32_t height);
/* restrict rasterisation + shading to pixel rows [row_begin, row_end) (screen-tile split, SURVEY 8e) */
int r3_set_scissor_rows(r3_ctx*, uint32_t row_begin, uint32_t row_end);

#ifdef __cplusplus
}
#endif
#endif /* REND3_B200_H */
