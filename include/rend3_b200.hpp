// rend3_b200.hpp — C++17 host-side mirror of rend3-routine's interface for the hot path, header-only, on top of the C ABI
// (include/rend3_b200.h).  The reference's host side is compiled code (Rust); no Rust toolchain exists in this image, so this is
// the native stand-in a C++ engine — or a Rust shim through the same C symbols (INTEGRATION.md) — would drive.  Names, argument
// meaning and call order follow the reference:
//
//   r3::GpuCuller::object_uniform_upload      rend3-routine/src/culling/culler.rs:427-529
//   r3::GpuSkinner::add_skinning_to_graph     skinning.rs:54-199 (node position base.rs:145)
//   r3::GpuCuller::add_culling_to_graph       culler.rs:682-713 (batch_objects, batching.rs:120-250, then cull, culler.rs:531-659)
//   r3::ForwardRoutine::add_forward_to_graph  forward.rs:192-315      r3::HiZRoutine::add_hi_z_to_graph   hi_z.rs:161-234
//   r3::TonemappingRoutine::add_to_graph      tonemapping.rs:108-147  r3::BaseRenderGraph::add_to_graph   base.rs:129-185
//
// What stays with the engine's managers is INPUT here, as the bytes they upload today: the object / material / light buffers,
// the PerCameraUniform header of every camera (culler.rs:484-505) and FrameUniforms (uniforms.rs:30-49).
// Error behaviour: the reference panics inside graph nodes (e.g. culler.rs:439,572); here every failure throws r3::Error carrying
// the C ABI's code and r3_last_error text — nothing unwinds across the C boundary.
#ifndef REND3_B200_HPP
#define REND3_B200_HPP

#include <array>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "rend3_b200.h"

namespace r3 {

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& what) : std::runtime_error(what), code(c) {}
};

enum class SampleCount : uint32_t { One = 1, Four = 4 };        // rend3-types SampleCount
enum class CullingSource { Predicted, Residual };               // forward.rs:134-142

// CameraSpecifier (rend3-routine/src/common/camera.rs): Viewport or Shadow(index); to_shader_index() is what the kernels see
struct CameraSpecifier {
    uint32_t index;
    static CameraSpecifier Viewport() { return {R3_CAMERA_VIEWPORT}; }
    static CameraSpecifier Shadow(uint32_t i) { return {i}; }
    bool is_shadow() const { return index != R3_CAMERA_VIEWPORT; }
    uint32_t to_shader_index() const { return index; }
};

// One shadow map of a directional light: its camera's PerCameraUniform header + the atlas viewport (directional.rs:24-119)
struct ShadowMap {
    r3_camera_header header;
    uint32_t offset[2];
    uint32_t size;
};

// What Renderer::evaluate_instructions leaves for the routines (renderer/eval.rs:9-181), as spans over the managers' bytes
struct EvalOutput {
    const r3_object* objects = nullptr; uint32_t n_slots = 0;                                   // object_manager.buffer::<M>()
    const uint64_t* material_key = nullptr; const uint8_t* sort_flags = nullptr; const float* location = nullptr;   // per slot
    const void* mesh_buffer = nullptr; uint64_t mesh_bytes = 0;
    const r3_material* materials = nullptr; uint32_t n_materials = 0;
    const r3_texture_desc* textures = nullptr; uint32_t n_textures = 0; const void* texels = nullptr; uint64_t texel_bytes = 0;
    const r3_texture_desc* skybox = nullptr; const void* skybox_texels = nullptr; uint64_t skybox_bytes = 0;     // SkyboxRoutine's cube map (null = none)
    const void* directional_lights = nullptr; uint64_t directional_bytes = 0; uint32_t shadow_target_size[2] = {0, 0};
    // the same lights as sources + atlas placements, in the light buffer's order, and the handedness: what
    // r3_set_directional_light_sources takes when the shadow cameras are evaluated on the device
    const r3_directional_light_source* directional_sources = nullptr; uint32_t n_directional_sources = 0; bool left_handed = true;
    // DirectionalLightChanges of this frame (DirectionalLightManager::update) for those sources, applied before their shadow cameras are
    // evaluated: in HOST memory or in DEVICE memory (producer ordered on the context's stream); both only enqueue work
    const r3_directional_light_change* directional_changes = nullptr; uint32_t n_directional_changes = 0;
    const r3_directional_light_change* d_directional_changes = nullptr; uint32_t n_d_directional_changes = 0;
    const void* point_lights = nullptr; uint64_t point_bytes = 0;
    // PointLightManager's handle table behind point_lights (records + live bytes, dead handles included): what
    // r3_set_point_light_sources takes when the point lights are evaluated on the device
    const r3_point_light_source* point_sources = nullptr; const uint8_t* point_live = nullptr; uint32_t n_point_handles = 0;
    std::vector<ShadowMap> shadows;
    r3_camera_header viewport{};              // PerCameraUniform header of the viewport camera for this target
    r3_frame_uniforms uniforms{};             // FrameUniforms::new
    float viewport_location[3] = {0, 0, 0};   // CameraState::location()
    // GPU skinning (skinning.rs:54-199): one record per skeleton + the global joint matrices; empty = no animated meshes this frame
    const r3_skinning_input* skinning_inputs = nullptr; uint32_t n_skeletons = 0; const float* joint_matrices = nullptr; uint32_t n_joints = 0;
    // instead: pose on the device and skin from the resident records and joint buffer (r3_set_animations / r3_set_skeletons /
    // r3_set_pose_jobs made before the frame); only enqueues work, so the frame stays one graph
    bool posed_skinning = false;
    // pose the animated nodes' objects on the device (r3_set_object_animations / r3_set_object_pose_jobs made before the frame):
    // transforms, world spheres and sort locations, written at the skinning node before any camera culls; only enqueues work
    bool posed_objects = false;
    // InternalObject::mesh_bounding_sphere per slot, (centre, radius) x n_slots (null = not uploaded: no object can be moved)
    const float* mesh_spheres = nullptr;
    // objects the application moved this frame (Renderer::set_object_transform in bulk): matrices (and slots, null = slots 0 .. n-1)
    // in DEVICE memory, their producer ordered on the context's stream; applied at the skinning node before posed_objects, enqueue only
    const uint32_t* d_moved_slots = nullptr; const float* d_moved_transforms = nullptr; uint32_t n_moved = 0;
    // objects that appear or disappear this frame (ObjectManager::add into a prepared slot / remove): presence bytes (and slots, null =
    // slots 0 .. n-1) in DEVICE memory, their producer ordered on the context's stream; applied at the skinning node before the moves
    const uint32_t* d_presence_slots = nullptr; const uint8_t* d_presence = nullptr; uint32_t n_presence = 0;
    // objects that change mesh or material this frame (ObjectManager::add with another mesh kind or material, within the set of
    // r3_set_object_variants made before the frame): choices (and slots, null = slots 0 .. n-1) in HOST memory (blocking) or in DEVICE
    // memory (enqueue only, producer ordered on the context's stream); applied at the skinning node before the presence and the moves
    const uint32_t* variant_slots = nullptr; const uint32_t* variant_choices = nullptr; uint32_t n_variant_switches = 0;
    const uint32_t* d_variant_slots = nullptr; const uint32_t* d_variant_choices = nullptr; uint32_t n_d_variant_switches = 0;
    // materials that change this frame (MaterialManager::update + evaluate's scatter of the stale records): records (and indices, null =
    // materials 0 .. n-1) in HOST memory (blocking, an index past the table grows it) or in DEVICE memory (enqueue only, records 16-byte
    // aligned, producer ordered on the context's stream); applied at the skinning node, before the shadow passes read the materials
    const uint32_t* material_indices = nullptr; const r3_material* material_records = nullptr; uint32_t n_material_updates = 0;
    const uint32_t* d_material_indices = nullptr; const r3_material* d_material_records = nullptr; uint32_t n_d_material_updates = 0;
    // skeletons posed by the application this frame (Renderer::set_skeleton_joint_matrices, or set_skeleton_joint_transforms when inverse
    // binds are given): writes and matrices in HOST memory (blocking) or in DEVICE memory (enqueue only, matrices 16-byte aligned, producer
    // ordered on the context's stream); applied at the skinning node after the posed_skinning pose, then r3_skin_posed skins from them
    const r3_joint_write* joint_writes = nullptr; uint32_t n_joint_writes = 0; const float* joint_mat4s = nullptr; uint32_t n_joint_mat4s = 0;
    const float* joint_inverse_binds = nullptr; uint32_t n_joint_inverse_binds = 0;
    const r3_joint_write* d_joint_writes = nullptr; uint32_t n_d_joint_writes = 0; const float* d_joint_mat4s = nullptr; uint32_t n_d_joint_mat4s = 0;
    const float* d_joint_inverse_binds = nullptr; uint32_t n_d_joint_inverse_binds = 0;
    // meshes that deform this frame (the set of r3_set_deformable_meshes rebuilt from new positions, its objects re-added): 3 floats per
    // vertex of the set, mesh after mesh, in HOST memory (blocking) or in DEVICE memory (enqueue only, 4-byte aligned, producer ordered on
    // the context's stream); applied first at the skinning node, so that a move wins the location and skinning reads the new positions
    const float* deform_positions = nullptr; uint64_t n_deform_floats = 0;
    const float* d_deform_positions = nullptr; uint64_t n_d_deform_floats = 0;
    // meshes whose topology changes this frame (the set of r3_set_remeshable_meshes rebuilt from new vertices and indices, its objects
    // re-added): the streams of r3_remesh_meshes at capacity strides, in HOST memory (blocking) or in DEVICE memory (enqueue only, 4-byte
    // aligned, producer ordered on the context's stream); applied where the deform is (a context holds one of the two sets), when
    // `counts` is set
    struct RemeshStreams {
        const uint32_t* counts = nullptr; const float* positions = nullptr; const uint32_t* indices = nullptr; const float* normals = nullptr;
        const float* tangents = nullptr; const float* uv0 = nullptr; const uint32_t* color0 = nullptr; uint64_t n_vertices = 0, n_indices = 0;
    };
    RemeshStreams remesh, d_remesh;
    // textures that change this frame (in rend3 added again and their materials updated): rectangles of stored bytes patched into the
    // table's and the skybox's levels, in HOST memory (blocking) or in DEVICE memory (enqueue only, regions 8-byte aligned, producer
    // ordered on the context's stream); applied before the first pass that samples them
    const r3_texture_region* texture_regions = nullptr; uint32_t n_texture_regions = 0; const void* texture_write_texels = nullptr; uint64_t texture_write_bytes = 0;
    const r3_texture_region* d_texture_regions = nullptr; uint32_t n_d_texture_regions = 0; const void* d_texture_write_texels = nullptr; uint64_t d_texture_write_bytes = 0;
};

struct BaseRenderGraphSettings {              // base.rs:95-98
    std::array<float, 4> ambient_color{0, 0, 0, 0};
    std::array<float, 4> clear_color{0, 0, 0, 0};
};

// Owns the device context (one per GPU); calls are externally serialised like rend3's data_core lock (graph.rs:265)
class Renderer {
public:
    explicit Renderer(int device) {
        const int rc = r3_ctx_create(device, &ctx_);
        if (rc != R3_OK) throw Error(rc, rc == R3_E_NO_DEVICE ? "no CUDA device (there is no CPU fallback)" : "r3_ctx_create failed");
    }
    ~Renderer() { if (ctx_) r3_ctx_destroy(ctx_); }
    Renderer(const Renderer&) = delete;
    Renderer& operator=(const Renderer&) = delete;
    r3_ctx* raw() const { return ctx_; }
    void check(int rc) const { if (rc != R3_OK) throw Error(rc, r3_last_error(ctx_)); }

    // renderer/eval.rs:157-181 — the buffers evaluate_instructions (re)uploads
    // device_shadow_cameras: the lights go up as sources (the frame evaluates their shadow cameras) instead of the light buffer;
    // device_point_lights: the point lights go up as the handle table (the frame evaluates them) instead of the evaluated buffer
    void upload_world(const EvalOutput& ev, bool device_shadow_cameras = false, bool device_point_lights = false) {
        check(r3_set_objects(ctx_, ev.objects, ev.n_slots));
        if (ev.material_key) check(r3_set_object_sort_info(ctx_, ev.material_key, ev.sort_flags, ev.location, ev.n_slots));
        if (ev.mesh_spheres) check(r3_set_object_mesh_spheres(ctx_, nullptr, ev.mesh_spheres, ev.n_slots));
        check(r3_set_mesh_buffer(ctx_, ev.mesh_buffer, ev.mesh_bytes));
        check(r3_set_textures(ctx_, ev.textures, ev.n_textures, ev.texels, ev.texel_bytes));
        check(r3_set_skybox(ctx_, ev.skybox, ev.skybox_texels, ev.skybox_bytes));
        check(r3_set_materials(ctx_, ev.materials, ev.n_materials));
        if (device_shadow_cameras)
            check(r3_set_directional_light_sources(ctx_, ev.directional_sources, ev.n_directional_sources, ev.shadow_target_size[0], ev.shadow_target_size[1],
                                                   ev.left_handed ? 1u : 0u));
        else
            check(r3_set_directional_lights(ctx_, ev.directional_lights, ev.directional_bytes, ev.shadow_target_size[0], ev.shadow_target_size[1]));
        if (device_point_lights) check(r3_set_point_light_sources(ctx_, ev.point_sources, ev.point_live, ev.n_point_handles));
        else check(r3_set_point_lights(ctx_, ev.point_lights, ev.point_bytes));
    }
    // Renderer::set_object_transform (object.rs:302-316) for n objects from host memory (slots == nullptr: slots 0 .. n-1); blocking
    void set_object_transforms(const uint32_t* slots, const float* mat4s, uint32_t n) { check(r3_set_object_transforms(ctx_, slots, mat4s, n)); }
    // ObjectManager::add into a prepared slot / remove for n slots from host memory (slots == nullptr: slots 0 .. n-1); blocking
    void set_objects_enabled(const uint32_t* slots, const uint8_t* enabled, uint32_t n) { check(r3_set_objects_enabled(ctx_, slots, enabled, n)); }
    void sync() { check(r3_sync(ctx_)); }

private:
    r3_ctx* ctx_ = nullptr;
};

class GpuCuller {   // culling/culler.rs:185-714
public:
    // object_uniform_upload: MV / MVP for every enabled slot + (fused here) the sphere-frustum filter of batch_objects
    void object_uniform_upload(Renderer& r, CameraSpecifier camera, const r3_camera_header& header) const {
        r.check(r3_object_uniform_upload(r.raw(), camera.to_shader_index(), &header, R3_CB_BAKE | R3_CB_CULL));
    }
    // add_culling_to_graph: batch_objects, then the per-triangle cull into the ping-pong CullingBuffers
    void add_culling_to_graph(Renderer& r, CameraSpecifier camera, const float viewport_location[3], uint32_t max_compute_workgroups_per_dimension = 65535) const {
        r.check(r3_batch_objects(r.raw(), camera.to_shader_index(), viewport_location, max_compute_workgroups_per_dimension));
        r.check(r3_cull(r.raw(), camera.to_shader_index(), nullptr, 0, nullptr, 0));
    }
};

class GpuSkinner {   // skinning.rs:54-199: add_skinning_to_graph — skinned positions / normals / tangents into the skeletons' overridden mesh ranges
public:
    void add_skinning_to_graph(Renderer& r, const EvalOutput& ev) const {
        if (ev.n_deform_floats) r.check(r3_deform_meshes(r.raw(), ev.deform_positions, ev.n_deform_floats));
        if (ev.n_d_deform_floats) r.check(r3_deform_meshes_device(r.raw(), ev.d_deform_positions, ev.n_d_deform_floats));
        if (const EvalOutput::RemeshStreams& s = ev.remesh; s.counts)
            r.check(r3_remesh_meshes(r.raw(), s.counts, s.positions, s.indices, s.normals, s.tangents, s.uv0, s.color0, s.n_vertices, s.n_indices));
        if (const EvalOutput::RemeshStreams& s = ev.d_remesh; s.counts)
            r.check(r3_remesh_meshes_device(r.raw(), s.counts, s.positions, s.indices, s.normals, s.tangents, s.uv0, s.color0, s.n_vertices, s.n_indices));
        if (ev.n_skeletons) r.check(r3_skin(r.raw(), ev.skinning_inputs, ev.n_skeletons, ev.joint_matrices, ev.n_joints));
        if (ev.n_variant_switches) r.check(r3_switch_object_variants(r.raw(), ev.variant_slots, ev.variant_choices, ev.n_variant_switches));
        if (ev.n_d_variant_switches) r.check(r3_switch_object_variants_device(r.raw(), ev.d_variant_slots, ev.d_variant_choices, ev.n_d_variant_switches));
        if (ev.n_presence) r.check(r3_set_objects_enabled_device(r.raw(), ev.d_presence_slots, ev.d_presence, ev.n_presence));
        if (ev.n_moved) r.check(r3_set_object_transforms_device(r.raw(), ev.d_moved_slots, ev.d_moved_transforms, ev.n_moved));
        if (ev.posed_objects) r.check(r3_pose_objects(r.raw()));
        if (ev.posed_skinning) r.check(r3_pose_skeletons(r.raw()));
        // the application's matrices after the clip's pose, so that an override (a ragdoll) wins
        if (ev.n_joint_writes)
            r.check(r3_set_joint_matrices(r.raw(), ev.joint_writes, ev.n_joint_writes, ev.joint_mat4s, ev.n_joint_mat4s, ev.joint_inverse_binds,
                                          ev.n_joint_inverse_binds));
        if (ev.n_d_joint_writes)
            r.check(r3_set_joint_matrices_device(r.raw(), ev.d_joint_writes, ev.n_d_joint_writes, ev.d_joint_mat4s, ev.n_d_joint_mat4s,
                                                 ev.d_joint_inverse_binds, ev.n_d_joint_inverse_binds));
        if (ev.posed_skinning || ev.n_joint_writes || ev.n_d_joint_writes) r.check(r3_skin_posed(r.raw()));
    }
};

class ForwardRoutine {   // forward.rs:85-315; opaque + cutout routines share one call, the blend routine has its own
public:
    void add_forward_to_graph(Renderer& r, CullingSource source) const { r.check(r3_forward_pass(r.raw(), source == CullingSource::Predicted ? 0 : 1)); }
    void add_shadow_to_graph(Renderer& r, uint32_t shadow_index, const ShadowMap& map) const {   // pbr_shadow_rendering, base.rs:366-396
        r.check(r3_shadow_pass(r.raw(), shadow_index, map.offset[0], map.offset[1], map.size));
    }
    void resolve(Renderer& r) const { r.check(r3_forward_resolve(r.raw())); }                     // fs_main of the winning fragments (+ SkyboxRoutine, base.rs:175)
    void add_transparent_to_graph(Renderer& r) const { r.check(r3_forward_blend(r.raw())); }       // pbr_forward_rendering_transparent
};

class HiZRoutine {
public:
    void add_hi_z_to_graph(Renderer& r) const { r.check(r3_hiz_build(r.raw())); }
};

class TonemappingRoutine {
public:
    void add_to_graph(Renderer& r, bool target_is_srgb) const { r.check(r3_tonemap(r.raw(), target_is_srgb ? 1 : 0)); }
};

// BaseRenderGraph::add_to_graph (base.rs:129-185): the node order of one frame, collapsed to a stream-ordered call sequence
class BaseRenderGraph {
public:
    GpuCuller gpu_culler;
    GpuSkinner gpu_skinner;
    ForwardRoutine forward;
    HiZRoutine hi_z;
    TonemappingRoutine tonemapping;
    bool submit_as_graph = false;             // record the frame and submit it as one CUDA graph launch (graph.rs:510: one submit per frame)
    // DirectionalLightManager::evaluate on the device (after Renderer::upload_world(ev, true)): the shadow cameras are evaluated around
    // this frame's viewport_location and culled from device memory; ev.shadows' headers are not read, only their atlas viewports
    bool device_shadow_cameras = false;
    // PointLightManager::evaluate on the device (after Renderer::upload_world(ev, ..., true)), right after the frame uniforms; add / update /
    // remove before it with r3_update_point_light_sources_device (enqueue only) or r3_update_point_light_sources
    bool device_point_lights = false;

    void add_to_graph(Renderer& r, const EvalOutput& ev, uint32_t width, uint32_t height, SampleCount samples, const BaseRenderGraphSettings& settings,
                      bool target_is_srgb = true) {
        r.check(r3_set_render_target(r.raw(), width, height, (uint32_t)samples, settings.clear_color.data()));
        if (submit_as_graph) r.check(r3_frame_begin(r.raw()));
        r.check(r3_clear_shadow_atlas(r.raw()));                                                     // base.rs:139
        r.check(r3_set_frame_uniforms(r.raw(), &ev.uniforms));                                       // :142
        if (ev.n_directional_changes) r.check(r3_update_directional_light_sources(r.raw(), ev.directional_changes, ev.n_directional_changes));
        if (ev.n_d_directional_changes)
            r.check(r3_update_directional_light_sources_device(r.raw(), ev.d_directional_changes, ev.n_d_directional_changes));
        if (device_shadow_cameras) r.check(r3_evaluate_shadow_cameras(r.raw(), ev.viewport_location));
        if (device_point_lights) r.check(r3_evaluate_point_lights(r.raw()));                       // renderer/eval.rs:180
        if (ev.n_texture_regions)
            r.check(r3_write_texture_regions(r.raw(), ev.texture_regions, ev.n_texture_regions, ev.texture_write_texels, ev.texture_write_bytes));
        if (ev.n_d_texture_regions)
            r.check(r3_write_texture_regions_device(r.raw(), ev.d_texture_regions, ev.n_d_texture_regions, ev.d_texture_write_texels, ev.d_texture_write_bytes));
        if (ev.n_material_updates) r.check(r3_update_materials(r.raw(), ev.material_indices, ev.material_records, ev.n_material_updates));
        if (ev.n_d_material_updates) r.check(r3_update_materials_device(r.raw(), ev.d_material_indices, ev.d_material_records, ev.n_d_material_updates));
        gpu_skinner.add_skinning_to_graph(r, ev);                                                    // :145 state.skinning — before any camera culls
        for (uint32_t i = 0; i < ev.shadows.size(); ++i) {                                          // :148
            if (device_shadow_cameras) r.check(r3_shadow_uniform_upload(r.raw(), i, ev.n_slots, R3_CB_BAKE | R3_CB_CULL));
            else gpu_culler.object_uniform_upload(r, CameraSpecifier::Shadow(i), ev.shadows[i].header);
        }
        for (uint32_t i = 0; i < ev.shadows.size(); ++i) gpu_culler.add_culling_to_graph(r, CameraSpecifier::Shadow(i), ev.viewport_location);     // :150
        for (uint32_t i = 0; i < ev.shadows.size(); ++i) forward.add_shadow_to_graph(r, i, ev.shadows[i]);                                         // :153
        gpu_culler.object_uniform_upload(r, CameraSpecifier::Viewport(), ev.viewport);               // :156
        r.check(r3_forward_begin(r.raw()));
        forward.add_forward_to_graph(r, CullingSource::Predicted);                                   // :159
        hi_z.add_hi_z_to_graph(r);                                                                   // :162
        gpu_culler.add_culling_to_graph(r, CameraSpecifier::Viewport(), ev.viewport_location);       // :169
        forward.add_forward_to_graph(r, CullingSource::Residual);                                    // :172
        forward.resolve(r);
        forward.add_transparent_to_graph(r);                                                         // :181
        tonemapping.add_to_graph(r, target_is_srgb);                                                 // :184
        if (submit_as_graph) r.check(r3_frame_end(r.raw()));
    }
};

}  // namespace r3
#endif
