/* r3_layouts.h — byte-exact std430 records shared by rend3's Rust managers and this library.
 *
 * These are the buffers the reference's managers already upload to wgpu; the C ABI in
 * rend3_b200.h consumes the very same bytes, so the Rust side needs no repacking.
 * Every struct cites the reference definition it mirrors (paths relative to the reference
 * repository root) and is checked with static_assert against the encase/std430 offsets.
 *
 * Plain C99 / C++11 / CUDA compatible.  No pointers, no torch types.
 */
#ifndef R3_LAYOUTS_H
#define R3_LAYOUTS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
#define R3_STATIC_ASSERT(c, m) static_assert(c, m)
#else
#define R3_STATIC_ASSERT(c, m) _Static_assert(c, m)
#endif

#define R3_INVALID_VERTEX 0x00FFFFFFu        /* rend3/shaders/vertex_attributes.wgsl:15 */
#define R3_CAMERA_VIEWPORT 0xFFFFFFFFu       /* CameraSpecifier::Viewport -> shadow_index u32::MAX (culler.rs:166-169) */
#define R3_ATTR_ABSENT 0xFFFFFFFFu           /* missing vertex attribute (managers/object.rs:263) */
#define R3_BATCH_SIZE 256u                   /* rend3-routine/src/culling/mod.rs:1 */
#define R3_WORKGROUP_SIZE 256u               /* rend3-routine/src/culling/mod.rs:2 */
#define R3_NO_PREVIOUS 0xFFFFFFFFu           /* batching.rs:226 */

/* PerCameraUniform.flags (culler.rs:151-156, structures.wgsl:64-72) */
#define R3_PCU_POSITIVE_AREA_VISIBLE 0x1u
#define R3_PCU_MULTISAMPLED 0x2u

/* PbrMaterial flags (rend3-routine/shaders/src/material.wgsl:1-15) */
#define R3_MAT_ALBEDO_ACTIVE 0x0001u
#define R3_MAT_ALBEDO_BLEND 0x0002u
#define R3_MAT_ALBEDO_VERTEX_SRGB 0x0004u
#define R3_MAT_BICOMPONENT_NORMAL 0x0008u
#define R3_MAT_SWIZZLED_NORMAL 0x0010u
#define R3_MAT_YDOWN_NORMAL 0x0020u
#define R3_MAT_AOMR_COMBINED 0x0040u
#define R3_MAT_AOMR_SWIZZLED_SPLIT 0x0080u
#define R3_MAT_AOMR_SPLIT 0x0100u
#define R3_MAT_AOMR_BW_SPLIT 0x0200u
#define R3_MAT_CC_GLTF_COMBINED 0x0400u
#define R3_MAT_CC_GLTF_SPLIT 0x0800u
#define R3_MAT_CC_BW_SPLIT 0x1000u
#define R3_MAT_UNLIT 0x2000u
#define R3_MAT_NEAREST 0x4000u

/* vertex attribute slot order of PbrMaterial::supported_attributes (pbr/material.rs:486-495) */
enum { R3_ATTR_POSITION = 0, R3_ATTR_NORMAL, R3_ATTR_TANGENT, R3_ATTR_UV0, R3_ATTR_UV1, R3_ATTR_COLOR0, R3_ATTR_COUNT };

/* ShaderObject<PbrMaterial> — rend3/src/managers/object.rs:23-36, structures_object.wgsl:3-12. stride 128 */
typedef struct r3_object {
    float transform[16];          /* @0   model->world, column major */
    float sphere_center[3];       /* @64  world-space bounding sphere (object.rs:269) */
    float sphere_radius;          /* @76 */
    uint32_t first_index;         /* @80  word index into the mesh buffer (object.rs:279) */
    uint32_t index_count;         /* @84 */
    uint32_t material_index;      /* @88 */
    uint32_t attr_offset[6];      /* @92  byte offsets into the mesh buffer, R3_ATTR_ABSENT if missing */
    uint32_t enabled;             /* @116 */
    uint32_t _pad[2];             /* @120 */
} r3_object;
R3_STATIC_ASSERT(sizeof(r3_object) == 128, "Object stride");
R3_STATIC_ASSERT(offsetof(r3_object, sphere_center) == 64, "sphere");
R3_STATIC_ASSERT(offsetof(r3_object, first_index) == 80, "first_index");
R3_STATIC_ASSERT(offsetof(r3_object, attr_offset) == 92, "attr offsets");
R3_STATIC_ASSERT(offsetof(r3_object, enabled) == 116, "enabled");

/* PerCameraUniform header — rend3-routine/src/culling/culler.rs:158-175, structures.wgsl:47-62.
 * `objects[]` (r3_object_matrices, stride 128) follows at byte 240. */
typedef struct r3_camera_header {
    float view[16];               /* @0 */
    float view_proj[16];          /* @64 */
    uint32_t shadow_index;        /* @128 R3_CAMERA_VIEWPORT for the viewport camera */
    uint32_t _pad0[3];
    float frustum[5][4];          /* @144 left,right,top,bottom,near: (abc, d) normalised (util/frustum.rs:96-145) */
    float resolution[2];          /* @224 */
    uint32_t flags;               /* @232 R3_PCU_* */
    uint32_t object_count;        /* @236 capacity of the object buffer (culler.rs:446-447) */
} r3_camera_header;
R3_STATIC_ASSERT(sizeof(r3_camera_header) == 240, "PerCameraUniform header");
R3_STATIC_ASSERT(offsetof(r3_camera_header, frustum) == 144, "frustum");
R3_STATIC_ASSERT(offsetof(r3_camera_header, resolution) == 224, "resolution");
R3_STATIC_ASSERT(offsetof(r3_camera_header, object_count) == 236, "object_count");

/* PerCameraUniformObjectData — culler.rs:177-183 */
typedef struct r3_object_matrices {
    float model_view[16];
    float model_view_proj[16];
} r3_object_matrices;
R3_STATIC_ASSERT(sizeof(r3_object_matrices) == 128, "PerCameraUniformObjectData");

/* ShaderObjectCullingInformation — culling/batching.rs:90-100 */
typedef struct r3_object_culling_info {
    uint32_t invocation_start;
    uint32_t invocation_end;
    uint32_t object_id;
    uint32_t region_id;
    uint32_t base_region_invocation;
    uint32_t local_region_id;
    uint32_t previous_global_invocation;
    uint32_t atomic_capable;
} r3_object_culling_info;
R3_STATIC_ASSERT(sizeof(r3_object_culling_info) == 32, "ObjectCullingInformation");

/* ShaderBatchData — culling/batching.rs:81-88 (#[align(256)] => 8448 bytes) */
typedef struct r3_batch_data {
    uint32_t total_objects;
    uint32_t total_invocations;
    uint32_t batch_base_invocation;
    r3_object_culling_info object_culling_information[256];
    uint32_t _pad[61];
} r3_batch_data;
R3_STATIC_ASSERT(sizeof(r3_batch_data) == 8448, "ShaderBatchData");
R3_STATIC_ASSERT(offsetof(r3_batch_data, object_culling_information) == 12, "batch table");

/* JobSubRegion + ShaderJobKey — culling/batching.rs:22-32 (host side only) */
typedef struct r3_region {
    uint32_t job_index;           /* batch this region's draw call binds (DrawCall::batch_index) */
    uint32_t bind_group_index;    /* TextureBindGroupIndex (DUMMY = 0 in the GpuDriven profile) */
    uint64_t material_key;
} r3_region;
R3_STATIC_ASSERT(sizeof(r3_region) == 16, "region");

/* IndirectCall — structures.wgsl:20-26 (20 bytes) */
typedef struct r3_indirect_call {
    uint32_t vertex_count;
    uint32_t instance_count;
    uint32_t base_index;
    int32_t vertex_offset;
    uint32_t base_instance;
} r3_indirect_call;
R3_STATIC_ASSERT(sizeof(r3_indirect_call) == 20, "IndirectCall");

/* FrameUniforms — rend3-routine/src/uniforms.rs:16-27, structures.wgsl:28-38 (uniform buffer, 496 B) */
typedef struct r3_frame_uniforms {
    float view[16];
    float view_proj[16];
    float origin_view_proj[16];
    float inv_view[16];
    float inv_view_proj[16];
    float inv_origin_view_proj[16];
    float frustum[5][4];          /* @384 */
    float ambient[4];             /* @464 */
    uint32_t resolution[2];       /* @480 */
    uint32_t _pad[2];
} r3_frame_uniforms;
R3_STATIC_ASSERT(sizeof(r3_frame_uniforms) == 496, "FrameUniforms");
R3_STATIC_ASSERT(offsetof(r3_frame_uniforms, ambient) == 464, "ambient");

/* ShaderDirectionalLight — rend3/src/managers/directional.rs:38-53; buffer = u32 count @0, array @16 */
typedef struct r3_directional_light {
    float view_proj[16];          /* @0 */
    float color[3];               /* @64 color*intensity */
    float _pad0;
    float direction[3];           /* @80 un-normalised (directional.rs:145) */
    float _pad1;
    float inv_resolution[2];      /* @96 1/atlas size */
    float atlas_offset[2];        /* @104 */
    float atlas_size[2];          /* @112 */
    float _pad2[2];
} r3_directional_light;
R3_STATIC_ASSERT(sizeof(r3_directional_light) == 128, "DirectionalLight");
R3_STATIC_ASSERT(offsetof(r3_directional_light, atlas_offset) == 104, "atlas_offset");

/* One directional light as the caller keeps it — rend3-types DirectionalLight (colour, intensity, direction, distance, resolution) —
 * plus its placement in the shadow atlas (directional/shadow_alloc.rs), in texels.  r3_set_directional_light_sources; host only. */
typedef struct r3_directional_light_source {
    float color[3];               /* @0 */
    float intensity;              /* @12 */
    float direction[3];           /* @16 un-normalised, as given */
    float distance;               /* @28 side of the shadow camera's box */
    uint32_t resolution;          /* @32 shadow map texels along a side (texel = distance / resolution) */
    uint32_t offset[2];           /* @36 atlas placement, texels */
    uint32_t size;                /* @44 */
} r3_directional_light_source;
R3_STATIC_ASSERT(sizeof(r3_directional_light_source) == 48, "DirectionalLight source");
R3_STATIC_ASSERT(offsetof(r3_directional_light_source, resolution) == 32, "resolution");

/* One DirectionalLightChange (rend3-types/src/lib.rs:1106-1121, applied field by field by update_from_changes, :232-238) for the light
 * at shadow index `index` of the current set: r3_update_directional_light_sources[_device].  A field is applied when its bit is in
 * `mask`.  There is no resolution bit: a new resolution re-packs the shadow atlas, which r3_set_directional_light_sources does. */
#define R3_DIR_CHANGE_COLOR 0x1u
#define R3_DIR_CHANGE_INTENSITY 0x2u
#define R3_DIR_CHANGE_DIRECTION 0x4u
#define R3_DIR_CHANGE_DISTANCE 0x8u
typedef struct r3_directional_light_change {
    uint32_t index;               /* @0  shadow index in the current set */
    uint32_t mask;                /* @4  R3_DIR_CHANGE_* */
    float color[3];               /* @8 */
    float intensity;              /* @20 */
    float direction[3];           /* @24 */
    float distance;               /* @36 */
    uint32_t _pad[2];             /* @40 */
} r3_directional_light_change;
R3_STATIC_ASSERT(sizeof(r3_directional_light_change) == 48, "DirectionalLightChange");
R3_STATIC_ASSERT(offsetof(r3_directional_light_change, mask) == 4, "mask");
R3_STATIC_ASSERT(offsetof(r3_directional_light_change, color) == 8, "color");
R3_STATIC_ASSERT(offsetof(r3_directional_light_change, intensity) == 20, "intensity");
R3_STATIC_ASSERT(offsetof(r3_directional_light_change, direction) == 24, "direction");
R3_STATIC_ASSERT(offsetof(r3_directional_light_change, distance) == 36, "distance");

/* ShaderPointLight — rend3/src/managers/point.rs:21-26; buffer = u32 count @0, array @16 */
typedef struct r3_point_light {
    float position[4];
    float color[3];
    float radius;
} r3_point_light;
R3_STATIC_ASSERT(sizeof(r3_point_light) == 32, "PointLight");

/* One point light as the caller keeps it — rend3-types PointLight (rend3-types/src/lib.rs:1124-1136), in its field order: one entry of
 * PointLightManager's handle table (r3_set_point_light_sources / r3_update_point_light_sources) */
typedef struct r3_point_light_source {
    float position[3];            /* @0 */
    float color[3];               /* @12 */
    float radius;                 /* @24 */
    float intensity;              /* @28 */
} r3_point_light_source;
R3_STATIC_ASSERT(sizeof(r3_point_light_source) == 32, "PointLight source");
R3_STATIC_ASSERT(offsetof(r3_point_light_source, color) == 12, "color");
R3_STATIC_ASSERT(offsetof(r3_point_light_source, radius) == 24, "radius");
R3_STATIC_ASSERT(offsetof(r3_point_light_source, intensity) == 28, "intensity");

/* GpuPoweredShaderWrapper<PbrMaterial> — managers/material.rs:25-29 + pbr/material.rs:526-543,
 * material.wgsl:21-57 (208 bytes) */
typedef struct r3_material {
    uint32_t textures[10];        /* @0 0 = none */
    uint32_t _pad0[2];
    float uv_transform0[3][4];    /* @48 mat3x3 columns padded to vec4 */
    float uv_transform1[3][4];    /* @96 */
    float albedo[4];              /* @144 */
    float emissive[3];            /* @160 */
    float roughness;              /* @172 */
    float metallic;               /* @176 */
    float reflectance;            /* @180 */
    float clear_coat;             /* @184 */
    float clear_coat_roughness;   /* @188 */
    float anisotropy;             /* @192 */
    float ambient_occlusion;      /* @196 */
    float alpha_cutout;           /* @200 */
    uint32_t flags;               /* @204 */
} r3_material;
R3_STATIC_ASSERT(sizeof(r3_material) == 208, "GpuMaterialData");
R3_STATIC_ASSERT(offsetof(r3_material, albedo) == 144, "albedo");
R3_STATIC_ASSERT(offsetof(r3_material, flags) == 204, "flags");

/* texture slots of r3_material.textures[] (material.wgsl:21-35): value = index into the texture table + 1, 0 = none */
enum { R3_TEX_ALBEDO = 0, R3_TEX_NORMAL, R3_TEX_ROUGHNESS, R3_TEX_METALLIC, R3_TEX_REFLECTANCE, R3_TEX_CLEAR_COAT, R3_TEX_CLEAR_COAT_ROUGHNESS,
       R3_TEX_EMISSIVE, R3_TEX_ANISOTROPY, R3_TEX_AMBIENT_OCCLUSION };

/* One entry of the bindless `textures` array (TextureManager<D2>, rend3/src/managers/texture.rs; binding opaque.wgsl:35):
 * a 2D texture with `mip_count` levels stored tightly one after the other (level l is max(w >> l, 1) x max(h >> l, 1))
 * starting at `byte_offset` of the texel blob handed to r3_set_textures. */
#define R3_TEXFMT_RGBA8_UNORM 0u
#define R3_TEXFMT_RGBA8_UNORM_SRGB 1u   /* rgb decoded to linear before filtering, alpha linear */
#define R3_TEXFMT_RGBA32_FLOAT 2u
#define R3_TEXFMT_R8_UNORM 3u           /* single channel (split AO / metallic / roughness maps): (r, 0, 0, 1) */
#define R3_TEXFMT_RG8_UNORM 4u          /* two channels (bicomponent normal maps): (r, g, 0, 1) */
/* Block-compressed formats (what rend3-gltf's ktx2 / dds loaders hand to add_texture_2d, rend3-gltf/src/lib.rs:1300-1335, 1455-1476,
 * 1556-1602): 4x4-texel blocks, row-major, level l stores ceil(w_l / 4) x ceil(h_l / 4) blocks of 8 (BC1, BC4) or 16 bytes.  The decode is
 * rule R11 of the oracle (oracle/r3_oracle_forward.inc): the ideal palette of the format as ONE IEEE division of two exact integers per
 * channel, e.g. BC1 code 2 red = (2 r0 + r1) / 93 with the 5-bit endpoints r0, r1.  BC7 is integer-exact by its specification (8-bit texels
 * from the interpolation ((64 - w) e0 + w e1 + 32) >> 6, then / 255); a block of the reserved mode reads (0, 0, 0, 0).  BC6H is not
 * implemented (r3_set_textures rejects it like any unknown format). */
#define R3_TEXFMT_BC1_RGBA_UNORM 5u
#define R3_TEXFMT_BC1_RGBA_UNORM_SRGB 6u
#define R3_TEXFMT_BC2_RGBA_UNORM 7u
#define R3_TEXFMT_BC2_RGBA_UNORM_SRGB 8u
#define R3_TEXFMT_BC3_RGBA_UNORM 9u
#define R3_TEXFMT_BC3_RGBA_UNORM_SRGB 10u
#define R3_TEXFMT_BC4_R_UNORM 11u        /* (r, 0, 0, 1) */
#define R3_TEXFMT_BC4_R_SNORM 12u
#define R3_TEXFMT_BC5_RG_UNORM 13u       /* (r, g, 0, 1) */
#define R3_TEXFMT_BC5_RG_SNORM 14u
#define R3_TEXFMT_BC7_RGBA_UNORM 15u
#define R3_TEXFMT_BC7_RGBA_UNORM_SRGB 16u
/* The other filterable uncompressed formats the ktx2 path can hand over (rend3-gltf/src/lib.rs:1195-1285).  Missing channels read (0, 0, 1);
 * snorm: max(v, -127) / 127; unorm16: v / 65535; Rgb10a2: 10-bit channels / 1023 from bit 0, alpha / 3; Bgra8: the bytes are b, g, r, a.
 * The integer (Uint / Sint) formats cannot be bound to a filtering sampler and are rejected. */
#define R3_TEXFMT_R8_SNORM 17u
#define R3_TEXFMT_RG8_SNORM 18u
#define R3_TEXFMT_RGBA8_SNORM 19u
#define R3_TEXFMT_BGRA8_UNORM 20u
#define R3_TEXFMT_BGRA8_UNORM_SRGB 21u
#define R3_TEXFMT_RGB10A2_UNORM 22u
#define R3_TEXFMT_R16_FLOAT 23u
#define R3_TEXFMT_RG16_FLOAT 24u
#define R3_TEXFMT_RGBA16_FLOAT 25u
#define R3_TEXFMT_R32_FLOAT 26u
#define R3_TEXFMT_RG32_FLOAT 27u
#define R3_TEXFMT_R16_UNORM 28u
#define R3_TEXFMT_RG16_UNORM 29u
#define R3_TEXFMT_RGBA16_UNORM 30u
#define R3_TEXFMT_COUNT 31u
#define R3_TEXFMT_IS_BLOCK(f) ((f) >= R3_TEXFMT_BC1_RGBA_UNORM && (f) <= R3_TEXFMT_BC7_RGBA_UNORM_SRGB)
#define R3_TEXFMT_BLOCK_BYTES(f) (((f) <= R3_TEXFMT_BC1_RGBA_UNORM_SRGB || (f) == R3_TEXFMT_BC4_R_UNORM || (f) == R3_TEXFMT_BC4_R_SNORM) ? 8u : 16u)
/* bytes per texel of an uncompressed format */
#define R3_TEXFMT_BPP(f) \
    ((f) == R3_TEXFMT_RGBA32_FLOAT ? 16u : \
     ((f) == R3_TEXFMT_RGBA16_FLOAT || (f) == R3_TEXFMT_RG32_FLOAT || (f) == R3_TEXFMT_RGBA16_UNORM) ? 8u : \
     ((f) == R3_TEXFMT_RG8_UNORM || (f) == R3_TEXFMT_RG8_SNORM || (f) == R3_TEXFMT_R16_FLOAT || (f) == R3_TEXFMT_R16_UNORM) ? 2u : \
     ((f) == R3_TEXFMT_R8_UNORM || (f) == R3_TEXFMT_R8_SNORM) ? 1u : 4u)
/* bytes of one w x h level */
#define R3_TEXFMT_LEVEL_BYTES(f, w, h) \
    (R3_TEXFMT_IS_BLOCK(f) ? (uint64_t)(((w) + 3u) / 4u) * (((h) + 3u) / 4u) * R3_TEXFMT_BLOCK_BYTES(f) : (uint64_t)(w) * (h) * R3_TEXFMT_BPP(f))
typedef struct r3_texture_desc {
    uint32_t width, height, mip_count, format;
    uint64_t byte_offset;
    uint64_t _reserved;
} r3_texture_desc;
R3_STATIC_ASSERT(sizeof(r3_texture_desc) == 32, "r3_texture_desc");

/* One rectangle of texels for r3_write_texture_regions[_device]: raw bytes in the target's storage format, copied into one level of one
 * texture of the table or one face of the skybox.  `texture` is a table index or R3_SKYBOX_FACE(f), f = 0..5 in the order +X -X +Y -Y +Z -Z.
 * x, y, width, height are texels of that level; the source rows (block rows for BC formats) start at src_offset and src_pitch apart. */
#define R3_SKYBOX_FACE(f) (0x80000000u | (f))
typedef struct r3_texture_region {
    uint64_t src_offset;          /* @0  bytes into the caller's source, a multiple of the element size */
    uint32_t texture;             /* @8  table index, or R3_SKYBOX_FACE(f) */
    uint32_t level;               /* @12 mip level of that texture / face */
    uint32_t x, y, width, height; /* @16 texels of that level */
    uint32_t src_pitch;           /* @32 bytes between consecutive source rows (block rows for BC formats) */
    uint32_t _reserved;           /* @36 0 */
} r3_texture_region;
R3_STATIC_ASSERT(sizeof(r3_texture_region) == 40, "r3_texture_region");
R3_STATIC_ASSERT(offsetof(r3_texture_region, texture) == 8, "texture");
R3_STATIC_ASSERT(offsetof(r3_texture_region, level) == 12, "level");
R3_STATIC_ASSERT(offsetof(r3_texture_region, x) == 16, "x");
R3_STATIC_ASSERT(offsetof(r3_texture_region, width) == 24, "width");
R3_STATIC_ASSERT(offsetof(r3_texture_region, src_pitch) == 32, "src_pitch");
R3_STATIC_ASSERT(offsetof(r3_texture_region, _reserved) == 36, "_reserved");

/* GpuSkinningInput — rend3-routine/src/skinning.rs:20-45, skinning.wgsl:3-26 (40 bytes, byte offsets into the mesh buffer,
 * R3_ATTR_ABSENT when an attribute is missing) */
typedef struct r3_skinning_input {
    uint32_t base_position_offset;
    uint32_t base_normal_offset;
    uint32_t base_tangent_offset;
    uint32_t joint_indices_offset;    /* [u16; 4] per vertex */
    uint32_t joint_weight_offset;     /* vec4<f32> per vertex */
    uint32_t updated_position_offset;
    uint32_t updated_normal_offset;
    uint32_t updated_tangent_offset;
    uint32_t joint_matrix_base_offset;
    uint32_t vertex_count;
} r3_skinning_input;
R3_STATIC_ASSERT(sizeof(r3_skinning_input) == 40, "GpuSkinningInput");

/* One mesh of a deformable set (r3_set_deformable_meshes): where MeshBuilder::build put its attributes and indices in the mesh buffer
 * (rend3-types/src/lib.rs:477-512, managers/mesh.rs:123-184) and which of them build computed from the positions.  r3_deform_meshes
 * writes the positions and recomputes what the flags name, as rebuilding the mesh from the new positions would. */
#define R3_DEFORM_LEFT_HANDED 0x1u           /* the renderer's handedness is Left: face normal edge1 x edge2 (else edge2 x edge1) */
#define R3_DEFORM_NORMALS 0x2u               /* built without normals: calculate_normals_for_buffers (lib.rs:662-702) */
#define R3_DEFORM_TANGENTS 0x4u              /* built without tangents and with uv0: calculate_tangents_for_buffers (lib.rs:784-836) */
typedef struct r3_deformable_mesh {
    uint32_t position_offset;     /* @0  byte offsets in the mesh buffer, R3_ATTR_ABSENT if missing */
    uint32_t normal_offset;       /* @4 */
    uint32_t tangent_offset;      /* @8 */
    uint32_t uv0_offset;          /* @12 */
    uint32_t first_index;         /* @16 the objects' first_index (a word index) and index_count; indices local to the mesh */
    uint32_t index_count;         /* @20 */
    uint32_t vertex_count;        /* @24 */
    uint32_t flags;               /* @28 R3_DEFORM_* */
} r3_deformable_mesh;
R3_STATIC_ASSERT(sizeof(r3_deformable_mesh) == 32, "r3_deformable_mesh");
R3_STATIC_ASSERT(offsetof(r3_deformable_mesh, uv0_offset) == 12, "uv0_offset");
R3_STATIC_ASSERT(offsetof(r3_deformable_mesh, first_index) == 16, "first_index");
R3_STATIC_ASSERT(offsetof(r3_deformable_mesh, flags) == 28, "flags");

/* One mesh of a remeshable set (r3_set_remeshable_meshes): a mesh whose topology changes every frame (an isosurface, a voxel chunk, a
 * fractured or cut mesh).  Its ranges in the mesh buffer are sized by the capacities; each remesh writes the first vertex_count entries
 * of every range and the first index_count indices, as MeshBuilder::build + MeshManager::add of the new vertices and indices would.
 * flags: R3_DEFORM_*, with the same meaning as in r3_deformable_mesh. */
typedef struct r3_remeshable_mesh {
    uint32_t position_offset;     /* @0  byte offsets in the mesh buffer, R3_ATTR_ABSENT if missing */
    uint32_t normal_offset;       /* @4 */
    uint32_t tangent_offset;      /* @8 */
    uint32_t uv0_offset;          /* @12 */
    uint32_t color0_offset;       /* @16 4 bytes per vertex */
    uint32_t first_index;         /* @20 the objects' first_index (a word index); indices local to the mesh */
    uint32_t index_capacity;      /* @24 */
    uint32_t vertex_capacity;     /* @28 */
    uint32_t flags;               /* @32 R3_DEFORM_* */
    uint32_t _pad[3];             /* @36 */
} r3_remeshable_mesh;
R3_STATIC_ASSERT(sizeof(r3_remeshable_mesh) == 48, "r3_remeshable_mesh");
R3_STATIC_ASSERT(offsetof(r3_remeshable_mesh, color0_offset) == 16, "color0_offset");
R3_STATIC_ASSERT(offsetof(r3_remeshable_mesh, first_index) == 20, "first_index");
R3_STATIC_ASSERT(offsetof(r3_remeshable_mesh, flags) == 32, "flags");

/* One prepared mesh + material of an object (r3_set_object_variants): what ObjectManager::add takes from the mesh kind and the material
 * (object.rs:267-284).  A switch writes these fields into the slot's record, moves mesh_sphere by the slot's transform and, when sort
 * info is set, takes material_key and sort_flags as the slot's key and flags bits 1-2. */
typedef struct r3_object_variant {
    uint32_t first_index;         /* @0  as r3_object (object.rs:279): word index of the mesh's indices */
    uint32_t index_count;         /* @4 */
    uint32_t material_index;      /* @8 */
    uint32_t attr_offset[6];      /* @12 byte offsets, R3_ATTR_ABSENT if missing */
    uint32_t sort_flags;          /* @36 bits 1-2 of r3_set_object_sort_info's flags (atomic, back to front); bit 0 (live) must be 0 */
    uint64_t material_key;        /* @40 Material::key */
    float mesh_sphere[4];         /* @48 InternalObject::mesh_bounding_sphere (centre, radius) */
} r3_object_variant;
R3_STATIC_ASSERT(sizeof(r3_object_variant) == 64, "r3_object_variant");
R3_STATIC_ASSERT(offsetof(r3_object_variant, index_count) == 4, "index_count");
R3_STATIC_ASSERT(offsetof(r3_object_variant, material_index) == 8, "material_index");
R3_STATIC_ASSERT(offsetof(r3_object_variant, attr_offset) == 12, "attr_offset");
R3_STATIC_ASSERT(offsetof(r3_object_variant, sort_flags) == 36, "sort_flags");
R3_STATIC_ASSERT(offsetof(r3_object_variant, material_key) == 40, "material_key");
R3_STATIC_ASSERT(offsetof(r3_object_variant, mesh_sphere) == 48, "mesh_sphere");
/* a run of variants a slot chooses from, e.g. one LOD chain: variants first .. first + count - 1 */
typedef struct r3_variant_group { uint32_t first, count; } r3_variant_group;
R3_STATIC_ASSERT(sizeof(r3_variant_group) == 8, "r3_variant_group");
/* per-mesh status of the last remesh (r3_readback_remesh_status): Mesh::validate's reasons (rend3-types/src/lib.rs:533-567), the first
 * that applies */
#define R3_REMESH_APPLIED 0u
#define R3_REMESH_OVER_CAPACITY 1u           /* vertex_count > vertex_capacity or index_count > index_capacity */
#define R3_REMESH_NOT_TRIANGLES 2u           /* index_count % 3 != 0 */
#define R3_REMESH_INDEX_OUT_OF_RANGE 3u      /* an index >= vertex_count */

/* ---- skeletal animation (rend3-anim/src/lib.rs:37-263, posed on the device by r3_pose_skeletons) */
#define R3_ANIM_NO_PARENT 0xFFFFFFFFu        /* the joint's node has no parent: global = local (lib.rs:253-255) */
#define R3_ANIM_PARENT_NOT_JOINT 0xFFFFFFFEu /* the parent node is not a joint of the skin: global = IDENTITY * local (lib.rs:249) */
#define R3_ANIM_ABSENT 0xFFFFFFFFu           /* r3_anim_track.times: the clip has no channel for this property */

/* Skin — rend3-gltf Skin (inverse_bind_matrices, joints) + PerSkinData.joint_nodes_topological_order (lib.rs:39-52): the skin's joints
 * are r3_anim_library.joints[first_joint, first_joint + joint_count), joint k of the skin being joints[first_joint + k] (k is the index
 * into inverse_bind_matrices and into the skeleton's joint matrices); order[first_joint, first_joint + joint_count) lists the skin's joint
 * indices in topological order, parents first. */
typedef struct r3_anim_skin {
    uint32_t first_joint;
    uint32_t joint_count;
} r3_anim_skin;
R3_STATIC_ASSERT(sizeof(r3_anim_skin) == 8, "r3_anim_skin");

/* One joint: its node's parent (node.parent through node_to_joint_idx, lib.rs:246), the node's bind pose
 * (local_transform.to_scale_rotation_translation(), lib.rs:227-228, decomposed on the host) and inverse_bind_matrices[k] (lib.rs:216). */
typedef struct r3_anim_joint {
    float bind_translation[3];    /* @0 */
    uint32_t parent;              /* @12 joint index within the skin, R3_ANIM_NO_PARENT or R3_ANIM_PARENT_NOT_JOINT */
    float bind_rotation[4];       /* @16 quaternion x, y, z, w */
    float bind_scale[3];          /* @32 */
    uint32_t _pad;
    float inverse_bind[16];       /* @48 column major */
} r3_anim_joint;
R3_STATIC_ASSERT(sizeof(r3_anim_joint) == 112, "r3_anim_joint");
R3_STATIC_ASSERT(offsetof(r3_anim_joint, parent) == 12, "parent");
R3_STATIC_ASSERT(offsetof(r3_anim_joint, bind_rotation) == 16, "bind_rotation");
R3_STATIC_ASSERT(offsetof(r3_anim_joint, inverse_bind) == 48, "inverse_bind");

/* AnimationChannel<T> (rend3-gltf/src/lib.rs:742-760): `count` key times at keys[times ..] and `value_count` values of 3 (translation,
 * scale) or 4 (rotation x, y, z, w) floats at keys[values ..].  times == R3_ANIM_ABSENT: no channel for this property. */
typedef struct r3_anim_track {
    uint32_t times;
    uint32_t values;
    uint32_t count;
    uint32_t value_count;
} r3_anim_track;
R3_STATIC_ASSERT(sizeof(r3_anim_track) == 16, "r3_anim_track");

/* AnimationChannels of one joint in one clip (Animation::channels, keyed by node).  animated == 0: the clip has no channel for the
 * joint's node, whose local matrix is then IDENTITY (lib.rs:219), not its bind pose. */
typedef struct r3_anim_channel {
    r3_anim_track translation;    /* @0 */
    r3_anim_track rotation;       /* @16 */
    r3_anim_track scale;          /* @32 */
    uint32_t animated;            /* @48 */
    uint32_t _pad[3];
} r3_anim_channel;
R3_STATIC_ASSERT(sizeof(r3_anim_channel) == 64, "r3_anim_channel");
R3_STATIC_ASSERT(offsetof(r3_anim_channel, animated) == 48, "animated");

/* Animation (rend3-gltf) bound to one skin, as AnimationData::from_gltf_scene binds them through node_to_joint_idx: channel k of the
 * clip, for joint k of the skin, is r3_anim_library.channels[first_channel + k]. */
typedef struct r3_anim_clip {
    uint32_t skin;
    uint32_t first_channel;
    float duration;               /* Animation::duration: time is clamped to [0, duration] (lib.rs:190) */
    uint32_t _pad;
} r3_anim_clip;
R3_STATIC_ASSERT(sizeof(r3_anim_clip) == 16, "r3_anim_clip");

/* One skin posed with `clip` at `time` (pose_animation_frame, per skin of the scene), its matrices written to
 * targets[first_target, first_target + target_count): every skeleton bound to the skin (PerSkinData::skeletons, lib.rs:259-261). */
typedef struct r3_pose_job {
    uint32_t clip;
    float time;
    uint32_t first_target;
    uint32_t target_count;
} r3_pose_job;
R3_STATIC_ASSERT(sizeof(r3_pose_job) == 16, "r3_pose_job");

/* A skeleton's range of the joint buffer (GpuSkinningInput::joint_matrix_base_offset) and its joint count: set_joint_matrices keeps the
 * first joint_count matrices (rend3/src/managers/skeleton.rs:151-162). */
typedef struct r3_pose_target {
    uint32_t joint_matrix_base_offset;
    uint32_t joint_count;
} r3_pose_target;
R3_STATIC_ASSERT(sizeof(r3_pose_target) == 8, "r3_pose_target");

/* One skeleton's joint matrices set by the application (Renderer::set_skeleton_joint_transforms / set_skeleton_joint_matrices,
 * rend3/src/renderer/mod.rs:302-337, managers/skeleton.rs:151-162), for r3_set_joint_matrices[_device].  The sources are indices, so
 * several writes may read one range (the armature's primitives posed alike; a crowd sharing one skin's inverse binds). */
typedef struct r3_joint_write {
    uint32_t joint_matrix_base_offset;  /* destination: the skeleton's GpuSkinningInput::joint_matrix_base_offset */
    uint32_t joint_count;               /* matrices written: the skeleton's joint count (set_joint_matrices keeps the first joint_count) */
    uint32_t first_matrix;              /* source: mat4s[first_matrix .. first_matrix + joint_count) */
    uint32_t first_inverse_bind;        /* source: inverse_binds[first_inverse_bind ..), read only when the call passes inverse binds */
} r3_joint_write;
R3_STATIC_ASSERT(sizeof(r3_joint_write) == 16, "r3_joint_write");

/* ---- object animation: the object-transform half of pose_animation_frame (rend3-anim/src/lib.rs:192-212, posed on the device by
 * r3_pose_objects).  Tracks are r3_anim_track over the key blob of r3_anim_object_library. */

/* A scene node that carries an object: its bind pose, local_transform.to_scale_rotation_translation() (lib.rs:194), decomposed on the
 * host.  A property without a track takes its bind value (lib.rs:196-199), not IDENTITY's. */
typedef struct r3_anim_node {
    float bind_translation[3];    /* @0 */
    uint32_t _pad0;
    float bind_rotation[4];       /* @16 quaternion x, y, z, w */
    float bind_scale[3];          /* @32 */
    uint32_t _pad1;
} r3_anim_node;
R3_STATIC_ASSERT(sizeof(r3_anim_node) == 48, "r3_anim_node");
R3_STATIC_ASSERT(offsetof(r3_anim_node, bind_rotation) == 16, "bind_rotation");
R3_STATIC_ASSERT(offsetof(r3_anim_node, bind_scale) == 32, "bind_scale");

/* One (node, AnimationChannels) entry of Animation::channels (lib.rs:192): the node's translation / rotation / scale tracks, each
 * possibly absent (times == R3_ANIM_ABSENT), and the node index into r3_anim_object_library.nodes. */
typedef struct r3_anim_node_channel {
    r3_anim_track translation;    /* @0 */
    r3_anim_track rotation;       /* @16 */
    r3_anim_track scale;          /* @32 */
    uint32_t node;                /* @48 */
    uint32_t _pad[3];
} r3_anim_node_channel;
R3_STATIC_ASSERT(sizeof(r3_anim_node_channel) == 64, "r3_anim_node_channel");
R3_STATIC_ASSERT(offsetof(r3_anim_node_channel, node) == 48, "node");

/* One Animation, with only the channels of nodes that carry objects: r3_anim_object_library.channels[first_channel,
 * first_channel + channel_count). */
typedef struct r3_anim_node_clip {
    uint32_t first_channel;
    uint32_t channel_count;
    float duration;               /* Animation::duration: time is clamped to [0, duration] (lib.rs:190) */
    uint32_t _pad;
} r3_anim_node_clip;
R3_STATIC_ASSERT(sizeof(r3_anim_node_clip) == 16, "r3_anim_node_clip");

/* One primitive of a posed node's object (object.inner.primitives, lib.rs:208-210): its object slot, the channel of the job's clip
 * that poses it (an index within the clip), and InternalObject::mesh_bounding_sphere (object.rs:268-270), which set_object_transform
 * moves to world space (object.rs:313).  Jobs are r3_pose_job records whose targets index these. */
typedef struct r3_object_pose_target {
    uint32_t slot;                /* @0 */
    uint32_t channel;             /* @4 */
    uint32_t _pad[2];
    float mesh_sphere_center[3];  /* @16 */
    float mesh_sphere_radius;     /* @28 */
} r3_object_pose_target;
R3_STATIC_ASSERT(sizeof(r3_object_pose_target) == 32, "r3_object_pose_target");
R3_STATIC_ASSERT(offsetof(r3_object_pose_target, mesh_sphere_center) == 16, "mesh_sphere_center");

#endif /* R3_LAYOUTS_H */
