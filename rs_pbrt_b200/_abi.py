"""ctypes mirror of include/pbrt_gpu.h and include/pbrt_host.h, and the loader of the in-tree library.

The loader FAILS LOUDLY when librs_pbrt_b200.so is missing: there is no Python or CPU fallback for
the hot path.
"""
import ctypes as C
import os
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
# RS_PBRT_B200_LIB: developer override to load an experiment build of the same library (tools/exp_variants.sh)
LIB_PATH = Path(os.environ.get("RS_PBRT_B200_LIB") or Path(__file__).resolve().parent / "librs_pbrt_b200.so")

PBRT_OK, PBRT_E_INVALID, PBRT_E_UNSUPPORTED, PBRT_E_CUDA, PBRT_E_NO_DEVICE = 0, -1, -2, -3, -4
PBRT_NO_MATERIAL = 0xFFFFFFFF
LIGHT_DIFFUSE_AREA, LIGHT_POINT, LIGHT_SPOT, LIGHT_DISTANT, LIGHT_INFINITE, LIGHT_GONIOMETRIC, LIGHT_PROJECTION = range(7)
MAT_MATTE, MAT_PLASTIC, MAT_METAL, MAT_MIRROR, MAT_GLASS, MAT_UBER, MAT_SUBSTRATE, MAT_TRANSLUCENT, MAT_MIX = range(9)
LIGHTS_UNIFORM, LIGHTS_POWER, LIGHTS_SPATIAL = 0, 1, 2
SAMPLER_SOBOL, SAMPLER_HALTON = 0, 1
INTEGRATOR_PATH, INTEGRATOR_AO, INTEGRATOR_DIRECT, INTEGRATOR_WHITTED = 0, 1, 2, 3
DIRECT_SAMPLE_ALL, DIRECT_SAMPLE_ONE = 0, 1
INSTANCING_REFERENCE, INSTANCING_FIXED = 0, 1
WRAP_REPEAT, WRAP_BLACK, WRAP_CLAMP = 0, 1, 2
MAP_UV, MAP_SPHERICAL, MAP_CYLINDRICAL, MAP_PLANAR = 0, 1, 2, 3
MESH_INSTANCE = 0xFFFFFFFF
RENDER_COUNT_WORK = 1
RENDER_SINGLE_STREAM = 2


class PbrtBvhNode(C.Structure):
    _fields_ = [("pmin", C.c_float * 3), ("pmax", C.c_float * 3), ("offset", C.c_int32), ("n_prims", C.c_uint16),
                ("axis", C.c_uint8), ("pad", C.c_uint8)]


class PbrtTri(C.Structure):
    _fields_ = [("v", C.c_uint32 * 3), ("mesh", C.c_uint32), ("material", C.c_uint32), ("area_light", C.c_int32)]


class PbrtMesh(C.Structure):
    _fields_ = [("p", C.POINTER(C.c_float)), ("n", C.POINTER(C.c_float)), ("s", C.POINTER(C.c_float)),
                ("uv", C.POINTER(C.c_float)), ("n_verts", C.c_uint32), ("reverse_orientation", C.c_uint8),
                ("transform_swaps_handedness", C.c_uint8), ("pad", C.c_uint8 * 2), ("alpha", C.c_uint32), ("shadow_alpha", C.c_uint32)]


class PbrtTexture(C.Structure):
    _fields_ = [("res", C.c_uint32 * 2), ("texels", C.POINTER(C.c_float)), ("channels", C.c_uint32), ("trilinear", C.c_uint32), ("max_anisotropy", C.c_float),
                ("wrap", C.c_uint32), ("su", C.c_float), ("sv", C.c_float), ("du", C.c_float), ("dv", C.c_float),
                ("mapping", C.c_uint32), ("map_m", C.c_float * 16), ("kind", C.c_uint32), ("value", C.c_float * 3), ("child", C.c_uint32 * 3)]


class PbrtMaterial(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("params", C.c_float * 24), ("tex", C.c_uint32 * 8), ("bump", C.c_uint32)]


class PbrtLight(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("L", C.c_float * 3), ("tri", C.c_uint32), ("two_sided", C.c_uint32), ("area", C.c_float),
                ("p", C.c_float * 3), ("w2l", C.c_float * 9), ("cos_total_width", C.c_float), ("cos_falloff_start", C.c_float),
                ("l2w", C.c_float * 9), ("env_res", C.c_uint32 * 2), ("env_texels", C.POINTER(C.c_float)), ("n_samples", C.c_uint32), ("fov", C.c_float)]


class PbrtInstance(C.Structure):
    _fields_ = [("root", C.c_uint32), ("identity", C.c_uint32), ("m", C.c_float * 16), ("m_inv", C.c_float * 16)]


class PbrtCamera(C.Structure):
    _fields_ = [("raster_to_camera", C.c_float * 16), ("camera_to_world", C.c_float * 16), ("lens_radius", C.c_float),
                ("focal_distance", C.c_float), ("shutter_open", C.c_float), ("shutter_close", C.c_float)]


class PbrtSceneDesc(C.Structure):
    _fields_ = [("nodes", C.POINTER(PbrtBvhNode)), ("n_nodes", C.c_uint32), ("tris", C.POINTER(PbrtTri)), ("n_tris", C.c_uint32),
                ("meshes", C.POINTER(PbrtMesh)), ("n_meshes", C.c_uint32), ("materials", C.POINTER(PbrtMaterial)),
                ("n_materials", C.c_uint32), ("lights", C.POINTER(PbrtLight)), ("n_lights", C.c_uint32), ("camera", PbrtCamera),
                ("world_bound", C.c_float * 6), ("instances", C.POINTER(PbrtInstance)), ("n_instances", C.c_uint32),
                ("textures", C.POINTER(PbrtTexture)), ("n_textures", C.c_uint32)]


class PbrtAnimatedTransform(C.Structure):
    _fields_ = [("start", C.c_float * 16), ("start_inv", C.c_float * 16), ("end", C.c_float * 16), ("end_inv", C.c_float * 16),
                ("start_time", C.c_float), ("end_time", C.c_float)]


class PbrtMotionDesc(C.Structure):
    _fields_ = [("camera", C.POINTER(PbrtAnimatedTransform)), ("instances", C.POINTER(PbrtAnimatedTransform))]


PBRT_CAMERA_PERSPECTIVE, PBRT_CAMERA_ORTHOGRAPHIC, PBRT_CAMERA_ENVIRONMENT = 0, 1, 2
PBRT_CAMERA_REALISTIC = 3
PBRT_MAX_LENS_ELEMENTS = 32


class PbrtCameraModel(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("full_resolution", C.c_uint32 * 2)]


class PbrtLensElement(C.Structure):
    _fields_ = [("curvature_radius", C.c_float), ("thickness", C.c_float), ("eta", C.c_float), ("aperture_radius", C.c_float)]


class PbrtRealisticLens(C.Structure):
    _fields_ = [("elements", C.POINTER(PbrtLensElement)), ("n_elements", C.c_uint32), ("exit_pupil_bounds", C.POINTER(C.c_float)),
                ("film_diagonal", C.c_float), ("simple_weighting", C.c_uint32)]


class PbrtRenderParams(C.Structure):
    _fields_ = [("sample_bounds", C.c_int32 * 4), ("cropped_pixel_bounds", C.c_int32 * 4), ("pixel_bounds", C.c_int32 * 4),
                ("filter_radius", C.c_float * 2), ("filter_table", C.c_float * 256), ("max_sample_luminance", C.c_float),
                ("spp", C.c_uint32), ("max_depth", C.c_uint32), ("rr_threshold", C.c_float), ("light_strategy", C.c_uint32),
                ("flags", C.c_uint32), ("sampler", C.c_uint32), ("sample_at_pixel_center", C.c_uint32),
                ("integrator", C.c_uint32), ("ao_samples", C.c_uint32), ("ao_cos_sample", C.c_uint32), ("instancing", C.c_uint32), ("direct_strategy", C.c_uint32)]


class PbrtStats(C.Structure):
    _fields_ = [("camera_rays", C.c_uint64), ("rays", C.c_uint64), ("closest_rays", C.c_uint64), ("shadow_rays", C.c_uint64),
                ("nodes_visited", C.c_uint64), ("tris_tested", C.c_uint64), ("light_tri_tests", C.c_uint64), ("ms_total", C.c_double),
                ("ms_trace", C.c_double), ("ms_shade", C.c_double), ("trace_launches", C.c_uint32), ("kernel_launches", C.c_uint32),
                ("shade_slots", C.c_uint64), ("shaded_vertices", C.c_uint64)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


GPU_SYMBOLS = ["pbrt_gpu_scene_create", "pbrt_gpu_scene_destroy", "pbrt_gpu_scene_bytes", "pbrt_gpu_render", "pbrt_gpu_render_device", "pbrt_gpu_render_samples",
               "pbrt_gpu_render_tiles_device", "pbrt_gpu_render_multi", "pbrt_gpu_host_register", "pbrt_gpu_host_unregister",
               "pbrt_gpu_intersect", "pbrt_gpu_intersect_p", "pbrt_gpu_last_error", "pbrt_gpu_abi_version", "pbrt_gpu_launch_count", "pbrt_gpu_kat_sincos", "pbrt_gpu_kat_acos_atan2", "pbrt_gpu_kat_log2",
               "pbrt_gpu_scene_create_motion", "pbrt_gpu_kat_animated_interpolate", "pbrt_gpu_scene_create_multi", "pbrt_gpu_scene_create_camera",
               "pbrt_gpu_scene_create_lens", "pbrt_gpu_kat_realistic_rays"]
HOST_SYMBOLS = ["pbrt_host_new", "pbrt_host_free", "pbrt_host_last_error", "pbrt_host_add_material", "pbrt_host_add_material_mix", "pbrt_host_add_trianglemesh",
                "pbrt_host_add_light_point", "pbrt_host_add_light_spot", "pbrt_host_add_light_distant", "pbrt_host_add_light_infinite", "pbrt_host_add_light_goniometric", "pbrt_host_add_light_projection", "pbrt_host_look_at", "pbrt_host_transform_times", "pbrt_host_camera_motion", "pbrt_host_motion_desc", "pbrt_host_film", "pbrt_host_camera_perspective", "pbrt_host_camera_orthographic", "pbrt_host_camera_environment", "pbrt_host_camera_model", "pbrt_host_camera_realistic", "pbrt_host_film_diagonal", "pbrt_host_lens", "pbrt_host_lens_exit_pupil", "pbrt_host_sampler_sobol", "pbrt_host_sampler_halton", "pbrt_host_integrator_ao", "pbrt_host_object_begin", "pbrt_host_object_end", "pbrt_host_object_instance", "pbrt_host_instancing", "pbrt_host_add_texture_image", "pbrt_host_material_texture", "pbrt_host_material_bump", "pbrt_host_mesh_alpha", "pbrt_host_texture_mapping", "pbrt_host_add_texture_constant", "pbrt_host_add_texture_scale", "pbrt_host_add_texture_mix", "pbrt_host_integrator_direct", "pbrt_host_integrator_whitted", "pbrt_host_light_samples",
                "pbrt_host_integrator_path", "pbrt_host_world_end", "pbrt_host_scene_desc", "pbrt_host_render_params", "pbrt_host_render",
                "pbrt_host_film_rgbw", "pbrt_host_film_clear", "pbrt_host_film_add_rgbw", "pbrt_host_film_rgb", "pbrt_host_write_image",
                "pbrt_host_bvh_build"]

_lib = None


def load():
    """Load the in-tree shared library and declare prototypes.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise RuntimeError(
            "%s is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` (nvcc, sm_90a). "
            "The PathIntegrator hot path has no CPU or Python fallback." % LIB_PATH)
    L = C.CDLL(str(LIB_PATH))
    bind(L)
    _lib = L
    return L


def bind(L):
    """Declare the prototypes of include/pbrt_gpu.h and include/pbrt_host.h on a loaded library."""
    fp, ip, u8p, u32p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint8), C.POINTER(C.c_uint32)
    vp = C.c_void_p
    L.pbrt_gpu_scene_create.argtypes = [C.POINTER(PbrtSceneDesc), C.c_int, C.POINTER(vp)]
    L.pbrt_gpu_scene_create_motion.argtypes = [C.POINTER(PbrtSceneDesc), C.POINTER(PbrtMotionDesc), C.c_int, C.POINTER(vp)]
    L.pbrt_gpu_scene_create_multi.argtypes = [C.POINTER(PbrtSceneDesc), C.POINTER(PbrtMotionDesc), C.POINTER(C.c_int), C.c_uint32, C.POINTER(vp)]
    L.pbrt_gpu_scene_create_camera.argtypes = [C.POINTER(PbrtSceneDesc), C.POINTER(PbrtMotionDesc), C.POINTER(PbrtCameraModel), C.POINTER(C.c_int), C.c_uint32,
                                               C.POINTER(vp)]
    L.pbrt_gpu_scene_create_lens.argtypes = [C.POINTER(PbrtSceneDesc), C.POINTER(PbrtMotionDesc), C.POINTER(PbrtCameraModel), C.POINTER(PbrtRealisticLens),
                                             C.POINTER(C.c_int), C.c_uint32, C.POINTER(vp)]
    L.pbrt_gpu_kat_realistic_rays.argtypes = [vp, C.c_uint32, fp, fp, fp, fp, fp, fp, fp, fp, fp, fp]
    L.pbrt_gpu_kat_animated_interpolate.argtypes = [C.c_int, C.POINTER(PbrtAnimatedTransform), C.c_uint32, fp, fp, fp]
    L.pbrt_gpu_scene_destroy.argtypes = [vp]
    L.pbrt_gpu_scene_destroy.restype = None
    L.pbrt_gpu_scene_bytes.argtypes = [vp]
    L.pbrt_gpu_scene_bytes.restype = C.c_uint64
    L.pbrt_gpu_render.argtypes = [vp, C.POINTER(PbrtRenderParams), ip, fp, C.POINTER(PbrtStats)]
    L.pbrt_gpu_render_device.argtypes = [vp, C.POINTER(PbrtRenderParams), ip, vp, vp, C.POINTER(PbrtStats)]
    L.pbrt_gpu_render_tiles_device.argtypes = [vp, C.POINTER(PbrtRenderParams), C.c_uint32, C.c_uint32, vp, vp, C.POINTER(PbrtStats)]
    L.pbrt_gpu_render_multi.argtypes = [C.POINTER(vp), C.c_uint32, C.POINTER(PbrtRenderParams), fp, C.POINTER(PbrtStats)]
    L.pbrt_gpu_host_register.argtypes = [vp, C.c_uint64]
    L.pbrt_gpu_host_unregister.argtypes = [vp]
    L.pbrt_gpu_render_samples.argtypes = [vp, C.POINTER(PbrtRenderParams), ip, fp, C.POINTER(PbrtStats)]
    L.pbrt_gpu_intersect.argtypes = [vp, C.c_uint32, fp, fp, fp, ip, fp, fp, C.POINTER(PbrtStats)]
    L.pbrt_gpu_intersect_p.argtypes = [vp, C.c_uint32, fp, fp, fp, u8p, C.POINTER(PbrtStats)]
    L.pbrt_gpu_last_error.restype = C.c_char_p
    L.pbrt_gpu_launch_count.restype = C.c_uint64
    L.pbrt_gpu_kat_sincos.argtypes = [C.c_int, C.c_uint32, fp, fp, fp]
    L.pbrt_gpu_kat_acos_atan2.argtypes = [C.c_int, C.c_uint32, fp, fp, fp, fp]
    L.pbrt_gpu_kat_log2.argtypes = [C.c_int, C.c_uint32, fp, fp]
    L.pbrt_host_new.restype = vp
    L.pbrt_host_free.argtypes = [vp]
    L.pbrt_host_free.restype = None
    L.pbrt_host_last_error.restype = C.c_char_p
    L.pbrt_host_add_material.argtypes = [vp, C.c_uint32, fp]
    L.pbrt_host_add_material_mix.argtypes = [vp, C.c_int, C.c_int, fp]
    L.pbrt_host_add_trianglemesh.argtypes = [vp, C.c_uint32, u32p, C.c_uint32, fp, fp, fp, fp, C.c_int, C.c_int, C.c_int, fp, C.c_int]
    L.pbrt_host_add_light_point.argtypes = [vp, fp, fp, fp]
    L.pbrt_host_add_light_spot.argtypes = [vp, fp, fp, fp, fp, C.c_float, C.c_float]
    L.pbrt_host_add_light_distant.argtypes = [vp, fp, fp, fp, fp]
    L.pbrt_host_add_light_infinite.argtypes = [vp, fp, fp, fp, C.c_uint32, C.c_uint32, fp, fp]
    L.pbrt_host_add_light_goniometric.argtypes = [vp, fp, fp, fp, C.c_uint32, C.c_uint32, fp, fp]
    L.pbrt_host_add_light_projection.argtypes = [vp, fp, fp, fp, C.c_uint32, C.c_uint32, C.c_float, fp, fp]
    L.pbrt_host_look_at.argtypes = [vp, fp, fp, fp]
    L.pbrt_host_transform_times.argtypes = [vp, C.c_float, C.c_float]
    L.pbrt_host_camera_motion.argtypes = [vp, fp]
    L.pbrt_host_motion_desc.argtypes = [vp]
    L.pbrt_host_motion_desc.restype = C.POINTER(PbrtMotionDesc)
    L.pbrt_host_film.argtypes = [vp, C.c_int, C.c_int, fp, C.c_char_p, C.c_float, C.c_float, C.c_float, C.c_float]
    L.pbrt_host_camera_perspective.argtypes = [vp, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, fp]
    L.pbrt_host_camera_orthographic.argtypes = [vp, C.c_float, C.c_float, C.c_float, C.c_float, fp]
    L.pbrt_host_camera_environment.argtypes = [vp, C.c_float, C.c_float]
    L.pbrt_host_camera_model.argtypes = [vp]
    L.pbrt_host_camera_model.restype = C.POINTER(PbrtCameraModel)
    L.pbrt_host_camera_realistic.argtypes = [vp, fp, C.c_int, C.c_float, C.c_float, C.c_int, C.c_float, C.c_float]
    L.pbrt_host_film_diagonal.argtypes = [vp, C.c_float]
    L.pbrt_host_lens.argtypes = [vp]
    L.pbrt_host_lens_exit_pupil.argtypes = [C.POINTER(PbrtLensElement), C.c_int, C.c_float, fp]
    L.pbrt_host_lens.restype = C.POINTER(PbrtRealisticLens)
    L.pbrt_host_sampler_sobol.argtypes = [vp, C.c_int]
    L.pbrt_host_sampler_halton.argtypes = [vp, C.c_int, C.c_int]
    L.pbrt_host_integrator_ao.argtypes = [vp, C.c_int, C.c_int]
    L.pbrt_host_object_begin.argtypes = [vp]
    L.pbrt_host_object_end.argtypes = [vp]
    L.pbrt_host_object_instance.argtypes = [vp, C.c_int, fp]
    L.pbrt_host_instancing.argtypes = [vp, C.c_uint32]
    L.pbrt_host_add_texture_image.argtypes = [vp, fp, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_float, C.c_uint32, C.c_float, C.c_int, C.c_float,
                                              C.c_float, C.c_float, C.c_float]
    L.pbrt_host_material_texture.argtypes = [vp, C.c_int, C.c_int, C.c_int]
    L.pbrt_host_material_bump.argtypes = [vp, C.c_int, C.c_int]
    L.pbrt_host_mesh_alpha.argtypes = [vp, C.c_int, C.c_int, C.c_int]
    L.pbrt_host_texture_mapping.argtypes = [vp, C.c_int, C.c_uint32, fp]
    L.pbrt_host_add_texture_constant.argtypes = [vp, fp, C.c_int]
    L.pbrt_host_add_texture_scale.argtypes = [vp, C.c_int, C.c_int]
    L.pbrt_host_add_texture_mix.argtypes = [vp, C.c_int, C.c_int, C.c_int]
    L.pbrt_host_integrator_direct.argtypes = [vp, C.c_uint32, C.c_uint32, ip]
    L.pbrt_host_integrator_whitted.argtypes = [vp, C.c_uint32, ip]
    L.pbrt_host_light_samples.argtypes = [vp, C.c_uint32]
    L.pbrt_host_integrator_path.argtypes = [vp, C.c_uint32, C.c_float, C.c_uint32, ip]
    L.pbrt_host_world_end.argtypes = [vp, C.c_uint32, C.c_int]
    L.pbrt_host_scene_desc.argtypes = [vp]
    L.pbrt_host_scene_desc.restype = C.POINTER(PbrtSceneDesc)
    L.pbrt_host_render_params.argtypes = [vp]
    L.pbrt_host_render_params.restype = C.POINTER(PbrtRenderParams)
    L.pbrt_host_render.argtypes = [vp, C.c_int, ip, C.POINTER(PbrtStats)]
    L.pbrt_host_film_rgbw.argtypes = [vp]
    L.pbrt_host_film_rgbw.restype = fp
    L.pbrt_host_film_clear.argtypes = [vp]
    L.pbrt_host_film_add_rgbw.argtypes = [vp, fp]
    L.pbrt_host_film_rgb.argtypes = [vp, fp]
    L.pbrt_host_write_image.argtypes = [vp, C.c_char_p]
    L.pbrt_host_bvh_build.argtypes = [fp, C.c_uint32, C.c_uint32, C.c_int, C.POINTER(PbrtBvhNode), u32p, u32p]
    return L
