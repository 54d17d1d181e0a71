"""ctypes binding of libezrt_b200.so -- exactly the entry points include/ezrt.h declares.

The library is the product; there is NO fallback: if it cannot be loaded (and cannot be
built because nvcc is absent) importing this module raises, and device entry points raise
EzrtError when no CUDA device is present.
"""
import ctypes as C
import os

from . import build as _build

c_float_p = C.POINTER(C.c_float)
c_int32_p = C.POINTER(C.c_int32)
c_uint32_p = C.POINTER(C.c_uint32)


class RenderParams(C.Structure):
    """struct ezrt_render_params (include/ezrt.h)."""
    _fields_ = [
        ("width", C.c_int32), ("height", C.c_int32), ("spp", C.c_int32), ("first_frame", C.c_uint32),
        ("max_bounce", C.c_int32), ("mode", C.c_int32),
        ("eye", C.c_float * 3), ("camera_rotate", C.c_float * 16), ("env_color", C.c_float * 3),
        ("traverse", C.c_int32), ("pipeline", C.c_int32), ("out_channels", C.c_int32),
        ("part_rank", C.c_int32), ("part_count", C.c_int32), ("frames_per_batch", C.c_int32),
        ("profile", C.c_int32), ("reserved", C.c_int32 * 3),
    ]


class AdaptiveParams(C.Structure):
    """struct ezrt_adaptive_params (include/ezrt.h)."""
    _fields_ = [("threshold", C.c_float), ("min_spp", C.c_int32), ("check_interval", C.c_int32), ("reserved", C.c_int32)]


class DenoiseParams(C.Structure):
    """struct ezrt_denoise_params (include/ezrt.h)."""
    _fields_ = [("iterations", C.c_int32), ("sigma_l", C.c_float), ("sigma_n", C.c_float), ("sigma_z", C.c_float), ("sigma_a", C.c_float),
                ("reserved", C.c_int32)]


class Medium(C.Structure):
    """struct ezrt_medium (include/ezrt.h)."""
    _fields_ = [("sigma_t", C.c_float), ("albedo", C.c_float * 3), ("g", C.c_float), ("box_min", C.c_float * 3), ("box_max", C.c_float * 3),
                ("reserved", C.c_int32)]


class Texture(C.Structure):
    """struct ezrt_texture (include/ezrt.h)."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("rgba", C.c_void_p), ("reserved", C.c_int32)]


class Volume(C.Structure):
    """struct ezrt_volume (include/ezrt.h)."""
    _fields_ = [("attenuation_color", C.c_float * 3), ("attenuation_distance", C.c_float), ("reserved", C.c_int32)]


class PunctualLight(C.Structure):
    """struct ezrt_punctual_light (include/ezrt.h)."""
    _fields_ = [("type", C.c_int32), ("position", C.c_float * 3), ("direction", C.c_float * 3), ("color", C.c_float * 3),
                ("intensity", C.c_float), ("inner_cone", C.c_float), ("outer_cone", C.c_float), ("reserved", C.c_int32)]


class Counters(C.Structure):
    """struct ezrt_counters (include/ezrt.h)."""
    _fields_ = [
        ("rays", C.c_uint64), ("primary_rays", C.c_uint64), ("bounce_rays", C.c_uint64), ("shadow_rays", C.c_uint64),
        ("samples", C.c_uint64), ("kernel_launches", C.c_uint64), ("device_ms", C.c_double),
        ("deferred_rays", C.c_uint64), ("node_visits", C.c_uint64), ("tri_tests", C.c_uint64), ("node_visits_96", C.c_uint64),
        ("node_bytes", C.c_uint64), ("tri_bytes", C.c_uint64),
    ]


# name -> (restype, argtypes); the list tests/test_abi.py checks against include/ezrt.h
SIGNATURES = {
    "ezrt_last_error": (C.c_char_p, []),
    "ezrt_version": (C.c_int, []),
    "ezrt_scene_create": (C.c_int, [C.c_int, c_float_p, C.c_int, c_float_p, C.c_int, c_float_p, c_float_p, C.c_int, C.c_int,
                                    C.c_int, C.POINTER(C.c_void_p)]),
    "ezrt_scene_destroy": (C.c_int, [C.c_void_p]),
    "ezrt_scene_set_medium": (C.c_int, [C.c_void_p, C.POINTER(Medium)]),
    "ezrt_scene_set_textures": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(Texture), c_float_p, c_int32_p]),
    "ezrt_scene_sample_textures": (C.c_int, [C.c_void_p, C.c_int, c_int32_p, c_float_p, c_float_p, c_float_p]),
    "ezrt_scene_set_emission_maps": (C.c_int, [C.c_void_p, c_int32_p]),
    "ezrt_scene_emission_lights": (C.c_int, [C.c_void_p, C.c_int, c_int32_p, c_float_p, c_float_p, C.POINTER(C.c_double)]),
    "ezrt_light_tree_build": (C.c_int, [C.c_int, c_float_p, c_float_p, C.c_int, c_float_p, c_uint32_p]),
    "ezrt_scene_light_tree": (C.c_int, [C.c_void_p, C.c_int, C.c_int, c_float_p, c_uint32_p]),
    "ezrt_scene_light_tree_eval": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, c_float_p, c_float_p, c_int32_p, c_int32_p, c_float_p]),
    "ezrt_scene_set_medium_grid": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, c_float_p]),
    "ezrt_scene_medium_grid": (C.c_int, [C.c_void_p, C.c_int, c_int32_p, c_float_p]),
    "ezrt_scene_set_volumes": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(Volume), c_int32_p]),
    "ezrt_scene_volumes": (C.c_int, [C.c_void_p, c_float_p]),
    "ezrt_scene_medium_eval": (C.c_int, [C.c_void_p, C.c_int, C.c_int, c_float_p, c_float_p, c_float_p, c_uint32_p, c_int32_p, c_float_p, c_uint32_p]),
    "ezrt_scene_sample_emission": (C.c_int, [C.c_void_p, C.c_int, c_int32_p, c_float_p, c_float_p]),
    "ezrt_scene_set_material_maps": (C.c_int, [C.c_void_p, c_int32_p, c_int32_p]),
    "ezrt_scene_sample_materials": (C.c_int, [C.c_void_p, C.c_int, c_int32_p, c_float_p, c_float_p]),
    "ezrt_scene_set_punctual_lights": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(PunctualLight)]),
    "ezrt_scene_punctual_lights": (C.c_int, [C.c_void_p, C.c_int, c_int32_p, c_float_p, c_float_p, C.POINTER(C.c_double)]),
    "ezrt_render": (C.c_int, [C.c_void_p, C.POINTER(RenderParams), c_float_p]),
    "ezrt_render_device": (C.c_int, [C.c_void_p, C.POINTER(RenderParams), C.c_void_p, C.c_void_p]),
    "ezrt_render_adaptive_device": (C.c_int, [C.c_void_p, C.POINTER(RenderParams), C.POINTER(AdaptiveParams), C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p]),
    "ezrt_render_adaptive": (C.c_int, [C.c_void_p, C.POINTER(RenderParams), C.POINTER(AdaptiveParams), c_float_p, c_int32_p, c_float_p]),
    "ezrt_render_aov_device": (C.c_int, [C.c_void_p, C.POINTER(RenderParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ezrt_render_aov": (C.c_int, [C.c_void_p, C.POINTER(RenderParams), c_float_p, c_float_p, c_float_p]),
    "ezrt_denoise_device": (C.c_int, [C.c_void_p, C.POINTER(DenoiseParams), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                      C.c_int, C.c_void_p, C.c_void_p]),
    "ezrt_denoise": (C.c_int, [C.c_void_p, C.POINTER(DenoiseParams), c_float_p, C.c_int, c_float_p, c_float_p, C.c_int, C.c_int, C.c_int,
                               c_float_p]),
    "ezrt_get_counters": (C.c_int, [C.c_void_p, C.POINTER(Counters)]),
    "ezrt_get_kernel_times": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_uint64)]),
    "ezrt_get_w8_phase_cycles": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64)]),
    "ezrt_get_w8_step_counts": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64)]),
    "ezrt_partition_pixels": (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "ezrt_partition_scatter": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "ezrt_partition_cache_clear": (C.c_int, [C.c_int]),
    "ezrt_host_sort_is_reference": (C.c_int, []),
    "ezrt_accel_build": (C.c_int, [C.c_int, c_float_p, C.c_int, C.c_int, C.c_int, c_int32_p, c_float_p, C.c_int, c_uint32_p, C.POINTER(C.c_double)]),
    "ezrt_partition_scatter_host": (C.c_int, [c_float_p, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "ezrt_trace_rays": (C.c_int, [C.c_void_p, C.c_int, c_float_p, c_float_p, C.c_int, C.c_int, C.c_int, c_int32_p, c_float_p,
                                  c_int32_p, c_int32_p, c_float_p, c_float_p]),
    "ezrt_scene_lights": (C.c_int, [C.c_void_p, C.c_int, c_int32_p, c_float_p, C.POINTER(C.c_double)]),
    "ezrt_scene_env_light": (C.c_int, [C.c_void_p, c_float_p, c_float_p, c_float_p, C.POINTER(C.c_double)]),
    "ezrt_occluded_rays": (C.c_int, [C.c_void_p, C.c_int, c_float_p, c_float_p, c_float_p, C.c_int, c_int32_p]),
    "ezrt_eval_brdf": (C.c_int, [C.c_int, C.c_int, C.c_int, c_float_p, c_float_p, c_float_p, c_float_p, c_float_p, c_float_p]),
    "ezrt_eval_bsdf": (C.c_int, [C.c_int, C.c_int, C.c_int, c_float_p, c_float_p, c_float_p, c_float_p, c_int32_p, c_float_p, c_float_p]),
    "ezrt_camera_rays": (C.c_int, [C.c_void_p, C.POINTER(RenderParams), C.c_int, c_uint32_p, c_uint32_p, c_uint32_p, c_float_p, c_float_p]),
    "ezrt_eval_math": (C.c_int, [C.c_int, C.c_int, C.c_int, c_float_p, c_float_p, c_float_p]),
    "ezrt_post_tonemap": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_float, C.c_void_p]),
    "ezrt_write_png": (C.c_int, [C.c_char_p, c_float_p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "ezrt_trilist_create": (C.c_void_p, []),
    "ezrt_trilist_destroy": (None, [C.c_void_p]),
    "ezrt_trilist_size": (C.c_int, [C.c_void_p]),
    "ezrt_transform_matrix": (None, [c_float_p, c_float_p, c_float_p, c_float_p]),
    "ezrt_trilist_read_obj": (C.c_int, [C.c_void_p, C.c_char_p, c_float_p, c_float_p, C.c_int]),
    "ezrt_trilist_read_obj_text": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, c_float_p, c_float_p, C.c_int]),
    "ezrt_trilist_append_encoded": (C.c_int, [C.c_void_p, c_float_p, C.c_int]),
    "ezrt_trilist_read_obj_textured": (C.c_int, [C.c_void_p, C.c_char_p, c_float_p, c_float_p, C.c_int, C.c_int32]),
    "ezrt_trilist_read_obj_textured_text": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, c_float_p, c_float_p, C.c_int, C.c_int32]),
    "ezrt_trilist_encode_texcoords": (C.c_int, [C.c_void_p, c_float_p, c_int32_p]),
    "ezrt_trilist_build_bvh": (C.c_int, [C.c_void_p, C.c_int, C.c_int]),
    "ezrt_trilist_node_count": (C.c_int, [C.c_void_p]),
    "ezrt_trilist_encode_triangles": (C.c_int, [C.c_void_p, c_float_p]),
    "ezrt_trilist_encode_nodes": (C.c_int, [C.c_void_p, c_float_p]),
    "ezrt_scene_file_load": (C.c_int, [C.c_char_p, C.c_void_p, c_float_p, C.c_char_p, C.c_size_t]),
    "ezrt_hdr_load": (C.c_int, [C.c_char_p, C.POINTER(C.c_int), C.POINTER(C.c_int), c_float_p]),
    "ezrt_hdr_cache": (C.c_int, [c_float_p, C.c_int, C.c_int, c_float_p]),
    "ezrt_hdr_cache_device": (C.c_int, [C.c_int, c_float_p, C.c_int, C.c_int, c_float_p, C.POINTER(C.c_double)]),
    "ezrt_camera_orbit": (None, [C.c_float, C.c_float, C.c_float, c_float_p, c_float_p]),
    "ezrt_camera_look_at": (C.c_int, [c_float_p, c_float_p, c_float_p, C.c_float, C.c_float, c_float_p]),
}


class EzrtError(RuntimeError):
    def __init__(self, code, message):
        super().__init__("ezrt error %d: %s" % (code, message))
        self.code = code


def _load():
    path = _build.PRODUCT_SO
    variant = os.environ.get("EZRT_LIB_VARIANT")
    if variant:  # experiment copy built by build.build_product(variant=..., defines=...)
        path = path.replace(".so", "_%s.so" % variant)
        return _bind(C.CDLL(path))
    # in-tree incremental build (no-op when the .so is newer than its sources); without nvcc a
    # prebuilt .so is used as is, and a missing one raises -- there is no CPU fallback
    # (ranks launched by torchrun never rebuild a library that exists: the launcher built/imported it first)
    if not os.path.exists(path) or (_build._nvcc() is not None and "RANK" not in os.environ and os.environ.get("EZRT_AUTO_BUILD", "1") != "0"):
        _build.build_product()
    return _bind(C.CDLL(path))


def _bind(lib):
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = restype
        fn.argtypes = argtypes
    return lib


lib = _load()
LIB_PATH = _build.PRODUCT_SO


def check(rc):
    if rc is not None and rc < 0:
        raise EzrtError(rc, (lib.ezrt_last_error() or b"").decode("utf-8", "replace"))
    return rc
