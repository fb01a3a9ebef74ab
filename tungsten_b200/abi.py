"""ctypes mirror of include/tgb200.h (the C ABI of libtgb200.so).

Field order and types must stay in lock-step with the header; tests/test_abi.py checks the struct
sizes against the values the library itself reports.
"""
import ctypes as C

ABI_VERSION = 3

TGB_OK, TGB_ERR_INVALID, TGB_ERR_UNSUPPORTED, TGB_ERR_NO_DEVICE, TGB_ERR_CUDA, TGB_ERR_ABORTED, TGB_ERR_OOM = \
    0, -1, -2, -3, -4, -5, -6

TEX_CONSTANT, TEX_CHECKER, TEX_BITMAP = 0, 1, 2
(BSDF_NULL, BSDF_LAMBERT, BSDF_ROUGH_CONDUCTOR, BSDF_ROUGH_DIELECTRIC, BSDF_PLASTIC, BSDF_ROUGH_PLASTIC,
 BSDF_SMOOTH_COAT, BSDF_CONDUCTOR, BSDF_DIELECTRIC, BSDF_MIRROR, BSDF_HAIR, BSDF_ROUGH_COAT) = range(12)
DIST_BECKMANN, DIST_PHONG, DIST_GGX = 0, 1, 2
PRIM_MESH, PRIM_QUAD, PRIM_CUBE, PRIM_INFINITE_SPHERE, PRIM_CURVES, PRIM_INFINITE_SPHERE_CAP, PRIM_SKYDOME = 0, 1, 2, 3, 4, 5, 6
CURVE_CYLINDER, CURVE_HALF_CYLINDER, CURVE_BCSDF_CYLINDER = 0, 1, 2
(FILTER_DIRAC, FILTER_BOX, FILTER_TENT, FILTER_GAUSSIAN, FILTER_MITCHELL, FILTER_CATMULL_ROM,
 FILTER_LANCZOS) = range(7)
# tgb200_bounce_probe's path-state record: word offsets (uint32 words; float fields are stored as their bits)
(BR_ORIGIN, BR_TMIN, BR_DIR, BR_STATUS, BR_THROUGHPUT, BR_BOUNCE, BR_EMISSION, BR_FLAGS, BR_PIXEL, BR_SEED, BR_SAMPLE,
 BR_DIMENSION, BR_PCG, BOUNCE_WORDS) = 0, 3, 4, 7, 8, 11, 12, 15, 16, 17, 18, 19, 20, 24

f32, u32, i32, u64 = C.c_float, C.c_uint32, C.c_int32, C.c_uint64
F3, F9 = f32*3, f32*9


class Texture(C.Structure):
    _fields_ = [("type", u32), ("value", F3), ("value2", F3), ("res_u", u32), ("res_v", u32),
                ("flags", u32), ("texels", C.POINTER(f32))]


class Bsdf(C.Structure):
    _fields_ = [("type", u32), ("albedo_tex", i32), ("distribution", u32), ("roughness_tex", i32),
                ("ior", f32), ("eta", F3), ("k", F3), ("thickness", f32), ("sigma_a", F3),
                ("substrate", i32), ("enable_refraction", u32),
                ("hair_scale_angle_deg", f32), ("hair_roughness", f32)]


class Vertex(C.Structure):
    _fields_ = [("pos", F3), ("normal", F3), ("uv", f32*2)]


class Triangle(C.Structure):
    _fields_ = [("v0", u32), ("v1", u32), ("v2", u32), ("material", i32)]


class Primitive(C.Structure):
    _fields_ = [("type", u32), ("emission_tex", i32),
                ("verts", C.POINTER(Vertex)), ("n_verts", u32),
                ("tris", C.POINTER(Triangle)), ("n_tris", u32),
                ("smooth", u32), ("bsdf_first", u32), ("bsdf_count", u32),
                ("base", F3), ("edge0", F3), ("edge1", F3),
                ("pos", F3), ("rot", F9), ("scale", F3),
                ("do_sample", u32),
                ("curve_nodes", C.POINTER(f32)), ("n_curve_nodes", u32),
                ("curve_segments", C.POINTER(u32)), ("n_curve_segments", u32),
                ("curve_mode", u32),
                ("cap_dir", F3), ("cap_cos", f32)]


class Camera(C.Structure):
    _fields_ = [("pos", F3), ("xform", F9), ("fov_deg", f32), ("res_x", u32), ("res_y", u32),
                ("filter", u32)]


class Settings(C.Structure):
    _fields_ = [("min_bounces", i32), ("max_bounces", i32), ("enable_light_sampling", u32),
                ("enable_two_sided_shading", u32), ("enable_consistency_checks", u32),
                ("use_sobol", u32), ("supplemental_mode", u32), ("device", i32),
                ("max_paths_in_flight", u32), ("n_devices", u32), ("devices", i32*8)]


class SceneDesc(C.Structure):
    _fields_ = [("abi_version", u32), ("camera", Camera), ("settings", Settings),
                ("primitives", C.POINTER(Primitive)), ("n_primitives", u32),
                ("bsdfs", C.POINTER(Bsdf)), ("n_bsdfs", u32),
                ("bsdf_slots", C.POINTER(u32)), ("n_bsdf_slots", u32),
                ("textures", C.POINTER(Texture)), ("n_textures", u32)]


class Tile(C.Structure):
    _fields_ = [("x", u32), ("y", u32), ("w", u32), ("h", u32), ("sampler_seed", u32)]


class Ray(C.Structure):
    _fields_ = [("o", F3), ("d", F3), ("tmin", f32), ("tmax", f32)]


class Hit(C.Structure):
    _fields_ = [("primitive", i32), ("prim_id", i32), ("t", f32), ("u", f32), ("v", f32),
                ("backside", u32)]


class Stats(C.Structure):
    _fields_ = [("samples", u64), ("rays", u64), ("hits", u64), ("kernel_launches", u64),
                ("trace_ms", C.c_double), ("trace_launches", u64), ("total_ms", C.c_double),
                ("path_rays", u64), ("shadow_rays", u64), ("shadow_ms", C.c_double), ("shadow_launches", u64),
                ("path_rays_traversed", u64), ("shadow_rays_traversed", u64),
                ("regen_ms", C.c_double), ("shade_ms", C.c_double), ("prep_ms", C.c_double), ("accum_ms", C.c_double),
                ("sort_ms", C.c_double), ("iterations", u64)]


class SampleRecord(C.Structure):
    _fields_ = [("sample_count", u32), ("next_sample_count", u32), ("sample_index", u32),
                ("adaptive_weight", f32), ("mean", f32), ("running_variance", f32)]


EXPORTS = [
    "tgb200_create", "tgb200_render_tiles", "tgb200_render_resident", "tgb200_clear_framebuffer",
    "tgb200_read_framebuffer", "tgb200_write_framebuffer", "tgb200_generate_work", "tgb200_render_adaptive", "tgb200_framebuffer_device_ptr", "tgb200_trace_closest", "tgb200_shard_tiles", "tgb200_pack_tiles", "tgb200_unpack_tiles",
    "tgb200_get_stats", "tgb200_set_profiling", "tgb200_set_stream", "tgb200_scene_info", "tgb200_reset_stats", "tgb200_bvh_selftest", "tgb200_hair_selftest", "tgb200_qbvh_selftest", "tgb200_shadow_walk_count", "tgb200_bsdf_probe", "tgb200_bsdf_sample_probe", "tgb200_light_probe",
    "tgb200_choose_light_probe", "tgb200_shadow_probe", "tgb200_bounce_probe", "tgb200_shade_variant", "tgb200_abort", "tgb200_clear_abort", "tgb200_destroy", "tgb200_last_error",
    "tgb200_abi_version",
]
