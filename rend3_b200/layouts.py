"""numpy mirrors of include/r3_layouts.h (std430 records shared with rend3's managers).

Each dtype has explicit offsets + itemsize so `.tobytes()` is byte-identical to what encase
writes on the Rust side.  tests/test_layouts.py cross-checks them against the C header by
compiling a sizeof/offsetof probe.
"""
import numpy as np

ATTR_ABSENT = 0xFFFFFFFF
CAMERA_VIEWPORT = 0xFFFFFFFF
INVALID_VERTEX = 0x00FFFFFF
NO_PREVIOUS = 0xFFFFFFFF
BATCH_SIZE = 256
WORKGROUP_SIZE = 256

PCU_POSITIVE_AREA_VISIBLE = 0x1
PCU_MULTISAMPLED = 0x2

MAT_ALBEDO_ACTIVE = 0x0001
MAT_ALBEDO_BLEND = 0x0002
MAT_ALBEDO_VERTEX_SRGB = 0x0004
MAT_BICOMPONENT_NORMAL = 0x0008
MAT_SWIZZLED_NORMAL = 0x0010
MAT_YDOWN_NORMAL = 0x0020
MAT_AOMR_COMBINED = 0x0040
MAT_AOMR_SWIZZLED_SPLIT = 0x0080
MAT_AOMR_SPLIT = 0x0100
MAT_AOMR_BW_SPLIT = 0x0200
MAT_CC_GLTF_COMBINED = 0x0400
MAT_CC_GLTF_SPLIT = 0x0800
MAT_CC_BW_SPLIT = 0x1000
MAT_UNLIT = 0x2000
MAT_NEAREST = 0x4000

f4, u4, i4 = np.float32, np.uint32, np.int32


def _dt(fields, itemsize):
    names, formats, offsets = zip(*fields)
    return np.dtype(dict(names=list(names), formats=list(formats), offsets=list(offsets), itemsize=itemsize))


OBJECT_DTYPE = _dt(
    [
        ("transform", (f4, 16), 0),
        ("sphere_center", (f4, 3), 64),
        ("sphere_radius", f4, 76),
        ("first_index", u4, 80),
        ("index_count", u4, 84),
        ("material_index", u4, 88),
        ("attr_offset", (u4, 6), 92),
        ("enabled", u4, 116),
    ],
    128,
)

CAMERA_HEADER_DTYPE = _dt(
    [
        ("view", (f4, 16), 0),
        ("view_proj", (f4, 16), 64),
        ("shadow_index", u4, 128),
        ("frustum", (f4, (5, 4)), 144),
        ("resolution", (f4, 2), 224),
        ("flags", u4, 232),
        ("object_count", u4, 236),
    ],
    240,
)

OBJECT_MATRICES_DTYPE = _dt([("model_view", (f4, 16), 0), ("model_view_proj", (f4, 16), 64)], 128)

CULLING_INFO_DTYPE = _dt(
    [
        ("invocation_start", u4, 0),
        ("invocation_end", u4, 4),
        ("object_id", u4, 8),
        ("region_id", u4, 12),
        ("base_region_invocation", u4, 16),
        ("local_region_id", u4, 20),
        ("previous_global_invocation", u4, 24),
        ("atomic_capable", u4, 28),
    ],
    32,
)

BATCH_DTYPE = _dt(
    [
        ("total_objects", u4, 0),
        ("total_invocations", u4, 4),
        ("batch_base_invocation", u4, 8),
        ("object_culling_information", (CULLING_INFO_DTYPE, 256), 12),
    ],
    8448,
)

REGION_DTYPE = _dt([("job_index", u4, 0), ("bind_group_index", u4, 4), ("material_key", np.uint64, 8)], 16)

INDIRECT_CALL_DTYPE = _dt(
    [
        ("vertex_count", u4, 0),
        ("instance_count", u4, 4),
        ("base_index", u4, 8),
        ("vertex_offset", i4, 12),
        ("base_instance", u4, 16),
    ],
    20,
)

FRAME_UNIFORMS_DTYPE = _dt(
    [
        ("view", (f4, 16), 0),
        ("view_proj", (f4, 16), 64),
        ("origin_view_proj", (f4, 16), 128),
        ("inv_view", (f4, 16), 192),
        ("inv_view_proj", (f4, 16), 256),
        ("inv_origin_view_proj", (f4, 16), 320),
        ("frustum", (f4, (5, 4)), 384),
        ("ambient", (f4, 4), 464),
        ("resolution", (u4, 2), 480),
    ],
    496,
)

DIRECTIONAL_LIGHT_DTYPE = _dt(
    [
        ("view_proj", (f4, 16), 0),
        ("color", (f4, 3), 64),
        ("direction", (f4, 3), 80),
        ("inv_resolution", (f4, 2), 96),
        ("atlas_offset", (f4, 2), 104),
        ("atlas_size", (f4, 2), 112),
    ],
    128,
)

POINT_LIGHT_DTYPE = _dt([("position", (f4, 4), 0), ("color", (f4, 3), 16), ("radius", f4, 28)], 32)

# r3_point_light_source: rend3-types PointLight, one entry of PointLightManager's handle table (r3_set_point_light_sources)
POINT_LIGHT_SOURCE_DTYPE = _dt([("position", (f4, 3), 0), ("color", (f4, 3), 12), ("radius", f4, 24), ("intensity", f4, 28)], 32)

# r3_directional_light_source: a DirectionalLight plus its atlas placement (r3_set_directional_light_sources)
LIGHT_SOURCE_DTYPE = _dt(
    [
        ("color", (f4, 3), 0),
        ("intensity", f4, 12),
        ("direction", (f4, 3), 16),
        ("distance", f4, 28),
        ("resolution", u4, 32),
        ("offset", (u4, 2), 36),
        ("size", u4, 44),
    ],
    48,
)

# r3_directional_light_change: one DirectionalLightChange for the light at a shadow index (r3_update_directional_light_sources[_device])
DIR_CHANGE_COLOR, DIR_CHANGE_INTENSITY, DIR_CHANGE_DIRECTION, DIR_CHANGE_DISTANCE = 1, 2, 4, 8
DIRECTIONAL_LIGHT_CHANGE_DTYPE = _dt([("index", u4, 0), ("mask", u4, 4), ("color", (f4, 3), 8), ("intensity", f4, 20), ("direction", (f4, 3), 24),
                                      ("distance", f4, 36)], 48)

MATERIAL_DTYPE = _dt(
    [
        ("textures", (u4, 10), 0),
        ("uv_transform0", (f4, (3, 4)), 48),
        ("uv_transform1", (f4, (3, 4)), 96),
        ("albedo", (f4, 4), 144),
        ("emissive", (f4, 3), 160),
        ("roughness", f4, 172),
        ("metallic", f4, 176),
        ("reflectance", f4, 180),
        ("clear_coat", f4, 184),
        ("clear_coat_roughness", f4, 188),
        ("anisotropy", f4, 192),
        ("ambient_occlusion", f4, 196),
        ("alpha_cutout", f4, 200),
        ("flags", u4, 204),
    ],
    208,
)

TEXTURE_DESC_DTYPE = _dt([("width", u4, 0), ("height", u4, 4), ("mip_count", u4, 8), ("format", u4, 12), ("byte_offset", np.dtype("<u8"), 16)], 32)

TEXFMT_RGBA8_UNORM, TEXFMT_RGBA8_UNORM_SRGB, TEXFMT_RGBA32_FLOAT, TEXFMT_R8_UNORM, TEXFMT_RG8_UNORM = 0, 1, 2, 3, 4
(TEXFMT_BC1_RGBA_UNORM, TEXFMT_BC1_RGBA_UNORM_SRGB, TEXFMT_BC2_RGBA_UNORM, TEXFMT_BC2_RGBA_UNORM_SRGB, TEXFMT_BC3_RGBA_UNORM, TEXFMT_BC3_RGBA_UNORM_SRGB,
 TEXFMT_BC4_R_UNORM, TEXFMT_BC4_R_SNORM, TEXFMT_BC5_RG_UNORM, TEXFMT_BC5_RG_SNORM, TEXFMT_BC7_RGBA_UNORM, TEXFMT_BC7_RGBA_UNORM_SRGB) = range(5, 17)   # 4x4 blocks, rule R11 (include/r3_layouts.h)
(TEXFMT_R8_SNORM, TEXFMT_RG8_SNORM, TEXFMT_RGBA8_SNORM, TEXFMT_BGRA8_UNORM, TEXFMT_BGRA8_UNORM_SRGB, TEXFMT_RGB10A2_UNORM, TEXFMT_R16_FLOAT, TEXFMT_RG16_FLOAT,
 TEXFMT_RGBA16_FLOAT, TEXFMT_R32_FLOAT, TEXFMT_RG32_FLOAT, TEXFMT_R16_UNORM, TEXFMT_RG16_UNORM, TEXFMT_RGBA16_UNORM) = range(17, 31)
TEXFMT_COUNT = 31


def texfmt_is_block(f: int) -> bool:
    """R3_TEXFMT_IS_BLOCK"""
    return TEXFMT_BC1_RGBA_UNORM <= f <= TEXFMT_BC7_RGBA_UNORM_SRGB


def texfmt_element_bytes(f: int) -> int:
    """Bytes of one stored element: the 4x4 block of a BC format (R3_TEXFMT_BLOCK_BYTES), else the texel (R3_TEXFMT_BPP)."""
    if texfmt_is_block(f):
        return 8 if f <= TEXFMT_BC1_RGBA_UNORM_SRGB or f in (TEXFMT_BC4_R_UNORM, TEXFMT_BC4_R_SNORM) else 16
    if f == TEXFMT_RGBA32_FLOAT:
        return 16
    if f in (TEXFMT_RGBA16_FLOAT, TEXFMT_RG32_FLOAT, TEXFMT_RGBA16_UNORM):
        return 8
    if f in (TEXFMT_RG8_UNORM, TEXFMT_RG8_SNORM, TEXFMT_R16_FLOAT, TEXFMT_R16_UNORM):
        return 2
    return 1 if f in (TEXFMT_R8_UNORM, TEXFMT_R8_SNORM) else 4


def texfmt_level_shape(f: int, width: int, height: int, level: int):
    """(texels wide, texels high, elements per row, rows) of mip `level` of a width x height texture; a BC row is a row of blocks."""
    w, h = max(width >> level, 1), max(height >> level, 1)
    return (w, h, (w + 3) // 4, (h + 3) // 4) if texfmt_is_block(f) else (w, h, w, h)


# r3_texture_region: one rectangle of texels for r3_write_texture_regions[_device]; `texture` is a table index or SKYBOX_FACE(f)
def SKYBOX_FACE(f: int) -> int:
    return 0x80000000 | int(f)


TEXTURE_REGION_DTYPE = _dt([("src_offset", np.dtype("<u8"), 0), ("texture", u4, 8), ("level", u4, 12), ("x", u4, 16), ("y", u4, 20),
                            ("width", u4, 24), ("height", u4, 28), ("src_pitch", u4, 32), ("_reserved", u4, 36)], 40)
(TEX_ALBEDO, TEX_NORMAL, TEX_ROUGHNESS, TEX_METALLIC, TEX_REFLECTANCE, TEX_CLEAR_COAT, TEX_CLEAR_COAT_ROUGHNESS, TEX_EMISSIVE, TEX_ANISOTROPY,
 TEX_AMBIENT_OCCLUSION) = range(10)

SKINNING_INPUT_DTYPE = _dt(
    [
        ("base_position_offset", u4, 0), ("base_normal_offset", u4, 4), ("base_tangent_offset", u4, 8), ("joint_indices_offset", u4, 12),
        ("joint_weight_offset", u4, 16), ("updated_position_offset", u4, 20), ("updated_normal_offset", u4, 24), ("updated_tangent_offset", u4, 28),
        ("joint_matrix_base_offset", u4, 32), ("vertex_count", u4, 36),
    ],
    40,
)

# skeletal animation (include/r3_layouts.h: rend3-anim/src/lib.rs:37-263)
ANIM_NO_PARENT = 0xFFFFFFFF
ANIM_PARENT_NOT_JOINT = 0xFFFFFFFE
ANIM_ABSENT = 0xFFFFFFFF
ANIM_SKIN_DTYPE = _dt([("first_joint", u4, 0), ("joint_count", u4, 4)], 8)
ANIM_JOINT_DTYPE = _dt([("bind_translation", (f4, 3), 0), ("parent", u4, 12), ("bind_rotation", (f4, 4), 16), ("bind_scale", (f4, 3), 32),
                        ("inverse_bind", (f4, 16), 48)], 112)
ANIM_TRACK_DTYPE = _dt([("times", u4, 0), ("values", u4, 4), ("count", u4, 8), ("value_count", u4, 12)], 16)
ANIM_CHANNEL_DTYPE = _dt([("translation", ANIM_TRACK_DTYPE, 0), ("rotation", ANIM_TRACK_DTYPE, 16), ("scale", ANIM_TRACK_DTYPE, 32),
                          ("animated", u4, 48)], 64)
ANIM_CLIP_DTYPE = _dt([("skin", u4, 0), ("first_channel", u4, 4), ("duration", f4, 8)], 16)
POSE_JOB_DTYPE = _dt([("clip", u4, 0), ("time", f4, 4), ("first_target", u4, 8), ("target_count", u4, 12)], 16)
POSE_TARGET_DTYPE = _dt([("joint_matrix_base_offset", u4, 0), ("joint_count", u4, 4)], 8)
# r3_set_joint_matrices[_device]: one skeleton's joint range and where its matrices (and inverse binds) are read from
JOINT_WRITE_DTYPE = _dt([("joint_matrix_base_offset", u4, 0), ("joint_count", u4, 4), ("first_matrix", u4, 8), ("first_inverse_bind", u4, 12)], 16)
# r3_set_deformable_meshes: where one mesh's attributes and indices are and what MeshBuilder::build computed (DEFORM_* flags)
DEFORMABLE_MESH_DTYPE = _dt([("position_offset", u4, 0), ("normal_offset", u4, 4), ("tangent_offset", u4, 8), ("uv0_offset", u4, 12),
                             ("first_index", u4, 16), ("index_count", u4, 20), ("vertex_count", u4, 24), ("flags", u4, 28)], 32)
DEFORM_LEFT_HANDED, DEFORM_NORMALS, DEFORM_TANGENTS = 0x1, 0x2, 0x4
# r3_set_remeshable_meshes: one mesh's capacity-sized ranges and how MeshBuilder::build made it (DEFORM_* flags)
REMESHABLE_MESH_DTYPE = _dt([("position_offset", u4, 0), ("normal_offset", u4, 4), ("tangent_offset", u4, 8), ("uv0_offset", u4, 12),
                             ("color0_offset", u4, 16), ("first_index", u4, 20), ("index_capacity", u4, 24), ("vertex_capacity", u4, 28),
                             ("flags", u4, 32)], 48)
# r3_set_object_variants: one prepared mesh + material of an object (what ObjectManager::add takes from the mesh kind and the material)
OBJECT_VARIANT_DTYPE = _dt([("first_index", u4, 0), ("index_count", u4, 4), ("material_index", u4, 8), ("attr_offset", (u4, 6), 12),
                            ("sort_flags", u4, 36), ("material_key", "<u8", 40), ("mesh_sphere", (f4, 4), 48)], 64)
VARIANT_GROUP_DTYPE = _dt([("first", u4, 0), ("count", u4, 4)], 8)
# r3_readback_object_variants: a slot the set does not list, or one not switched since the set was made
VARIANT_NONE = 0xFFFFFFFF
# r3_readback_remesh_status: Mesh::validate's reasons, the first that applies
REMESH_APPLIED, REMESH_OVER_CAPACITY, REMESH_NOT_TRIANGLES, REMESH_INDEX_OUT_OF_RANGE = 0, 1, 2, 3
# object animation (r3_set_object_animations / r3_set_object_pose_jobs); jobs are POSE_JOB_DTYPE records
ANIM_NODE_DTYPE = _dt([("bind_translation", (f4, 3), 0), ("bind_rotation", (f4, 4), 16), ("bind_scale", (f4, 3), 32)], 48)
ANIM_NODE_CHANNEL_DTYPE = _dt([("translation", ANIM_TRACK_DTYPE, 0), ("rotation", ANIM_TRACK_DTYPE, 16), ("scale", ANIM_TRACK_DTYPE, 32),
                               ("node", u4, 48)], 64)
ANIM_NODE_CLIP_DTYPE = _dt([("first_channel", u4, 0), ("channel_count", u4, 4), ("duration", f4, 8)], 16)
OBJECT_POSE_TARGET_DTYPE = _dt([("slot", u4, 0), ("channel", u4, 4), ("mesh_sphere_center", (f4, 3), 16), ("mesh_sphere_radius", f4, 28)], 32)
