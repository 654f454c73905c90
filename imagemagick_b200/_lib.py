"""ctypes binding of libmagickb200.so (include/magick_b200.h).

There is no Python / CPU fallback: if the shared library is missing the import of
the operators fails loudly (build it with ``python -m imagemagick_b200.build``).
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

LIB_PATH = Path(__file__).resolve().parent / "lib" / "libmagickb200.so"

OK, EINVAL, ENODEVICE, ECUDA, ENOMEM, EUNSUPPORTED = 0, -1, -2, -3, -4, -5


class MagickB200Error(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"libmagickb200 error {code}: {message}")
        self.code = code


class KernelInfoStruct(C.Structure):
    pass


KernelInfoStruct._fields_ = [
    ("type", C.c_int),
    ("width", C.c_size_t),
    ("height", C.c_size_t),
    ("x", C.c_long),
    ("y", C.c_long),
    ("values", C.POINTER(C.c_double)),
    ("minimum", C.c_double),
    ("maximum", C.c_double),
    ("negative_range", C.c_double),
    ("positive_range", C.c_double),
    ("angle", C.c_double),
    ("next", C.POINTER(KernelInfoStruct)),
]
KernelPtr = C.POINTER(KernelInfoStruct)

_f = C.POINTER(C.c_float)
_sz, _i, _d, _l, _vp = C.c_size_t, C.c_int, C.c_double, C.c_long, C.c_void_p

# name -> (restype, argtypes); this table is also what tests use to check that every
# symbol the header declares is exported.
PROTOTYPES = {
    "mb200_device_count": (_i, []),
    "mb200_set_device": (_i, [_i]),
    "mb200_last_error": (C.c_char_p, []),
    "mb200_version": (C.c_char_p, []),
    "mb200_launch_count": (C.c_ulonglong, []),
    "mb200_synchronize": (_i, [_vp]),
    "mb200_malloc": (_i, [C.POINTER(_vp), _sz]),
    "mb200_free": (_i, [_vp]),
    "mb200_malloc_host": (_i, [C.POINTER(_vp), _sz]),
    "mb200_free_host": (_i, [_vp]),
    "mb200_upload": (_i, [_vp, _vp, _sz, _vp]),
    "mb200_download": (_i, [_vp, _vp, _sz, _vp]),
    "mb200_trim": (_i, [_sz]),
    "mb200_probe_fp64_fma_rate": (_i, [C.POINTER(_d)]),
    "mb200_set_option": (_i, [C.c_char_p, _i]),
    "mb200_get_option": (_i, [C.c_char_p, C.POINTER(_i)]),
    "mb200_cache_attach": (_i, [_vp, _sz, _i]),
    "mb200_cache_detach": (_i, [_vp]),
    "mb200_cache_sync": (_i, [_vp]),
    "mb200_cache_host_written": (_i, [_vp]),
    "mb200_cache_resident": (_i, [_vp]),
    "mb200_cache_set_lazy": (_i, [_i]),
    "mb200_cache_stats": (None, [C.POINTER(C.c_ulonglong)]),
    "mb200_copy_threads": (_i, []),
    "mb200_acquire_kernel_info": (KernelPtr, [C.c_char_p]),
    "mb200_acquire_kernel_builtin": (KernelPtr, [_i, _d, _d, _d, _d]),
    "mb200_clone_kernel_info": (KernelPtr, [KernelPtr]),
    "mb200_destroy_kernel_info": (KernelPtr, [KernelPtr]),
    "mb200_scale_kernel_info": (None, [KernelPtr, _d, _i]),
    "mb200_optimal_kernel_width_1d": (_sz, [_d, _d]),
    "mb200_optimal_kernel_width_2d": (_sz, [_d, _d]),
    "mb200_resize_contributions": (_l, [_i, _sz, _sz, _d, C.POINTER(_l), C.POINTER(_i), C.POINTER(_d), _sz]),
    "mb200_resize_filter_weight": (_d, [_i, _d]),
    "mb200_resize_filter_weight_ex": (_d, [_i, _vp, _d]),
    "mb200_resize_filter_support_ex": (_d, [_i, _vp]),
    "mb200_resize_contributions_ex": (_l, [_i, _vp, _sz, _sz, _d, C.POINTER(_l), C.POINTER(_i), C.POINTER(_d), _sz]),
    "mb200_resize_filter_support": (_d, [_i]),
    "mb200_morphology_primitive_dev": (_i, [_vp, _vp, _sz, _sz, _i, _i, KernelPtr, _d, C.POINTER(C.c_longlong), _vp]),
    "mb200_morphology_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _i, _l, KernelPtr, _d, _vp]),
    "mb200_morphology_direct_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _i, KernelPtr, _vp]),
    "mb200_distort_image_dev": (_i, [_vp, _sz, _sz, _i, _vp, _vp, _vp, _vp]),
    "mb200_distort_image": (_i, [_vp, _sz, _sz, _i, _vp, _vp, _vp]),
    "mb200_distort_plan": (_i, [_i, _vp, _sz, _i, _sz, _sz, _l, _l, _vp, _d, _vp]),
    "mb200_rotate_plan": (_i, [_d, _sz, _sz, _l, _l, _vp]),
    "mb200_geometry_plan": (_i, [_i, _sz, _sz, _vp, _vp, _vp]),
    "mb200_geometry_image_dev": (_i, [_vp, _sz, _sz, _i, _vp, _vp, _vp]),
    "mb200_geometry_image": (_i, [_vp, _sz, _sz, _i, _vp, _vp]),
    "mb200_bounding_box_from_rows": (_i, [_vp, _sz, _sz, _i, _vp, _vp]),
    "mb200_trim_plan": (_i, [_sz, _sz, _vp, _vp, _i, _vp, _vp]),
    "mb200_bounding_box_dev": (_i, [_vp, _sz, _sz, _i, _vp, _vp, _vp, _vp]),
    "mb200_bounding_box": (_i, [_vp, _sz, _sz, _i, _vp, _vp, _vp]),
    "mb200_resample_filter_lut": (_i, [_i, _vp, _vp, _vp]),
    "mb200_convolve_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, KernelPtr, _vp]),
    "mb200_blur_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d, _vp]),
    "mb200_gaussian_blur_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d, _vp]),
    "mb200_unsharp_mask_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d, _d, _d, _vp]),
    "mb200_resize_image_dev": (_i, [_vp, _sz, _sz, _i, _vp, _sz, _sz, _i, _vp]),
    "mb200_resize_image_ex_dev": (_i, [_vp, _sz, _sz, _i, _vp, _sz, _sz, _i, _vp, _vp]),
    "mb200_resize_image_ex": (_i, [_vp, _sz, _sz, _i, _vp, _sz, _sz, _i, _vp]),
    "mb200_transform_colorspace_dev": (_i, [_vp, _sz, _sz, _i, _i, _i, _vp]),
    "mb200_transform_colorspace_ex_dev": (_i, [_vp, _sz, _sz, _i, _i, _i, _vp, _vp]),
    "mb200_blur_image": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d]),
    "mb200_gaussian_blur_image": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d]),
    "mb200_convolve_image": (_i, [_vp, _vp, _sz, _sz, _i, KernelPtr]),
    "mb200_morphology_image": (_i, [_vp, _vp, _sz, _sz, _i, _i, _l, KernelPtr, _d]),
    "mb200_morphology_direct_image": (_i, [_vp, _vp, _sz, _sz, _i, _i, KernelPtr]),
    "mb200_unsharp_mask_image": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d, _d, _d]),
    "mb200_resize_image": (_i, [_vp, _sz, _sz, _i, _vp, _sz, _sz, _i]),
    "mb200_transform_colorspace": (_i, [_vp, _sz, _sz, _i, _i, _i]),
    "mb200_transform_colorspace_ex": (_i, [_vp, _sz, _sz, _i, _i, _i, _vp]),
    "mb200_colorspace_channels": (_i, [_i, _i]),
    "mb200_transform_colorspace_layout_dev": (_i, [_vp, _i, _vp, _i, _sz, _sz, _i, _i, _vp, _vp]),
    "mb200_transform_colorspace_layout": (_i, [_vp, _i, _vp, _i, _sz, _sz, _i, _i, _vp]),
    "mb200_log_colorspace_table": (_i, [_i, _vp, _vp]),
    "mb200_ycc_table": (_i, [_vp]),
    "mb200_sharpen_kernel": (KernelPtr, [_d, _d]),
    "mb200_edge_kernel": (KernelPtr, [_d]),
    "mb200_restore_channels_dev": (_i, [_vp, _vp, _sz, _sz, _i, C.c_uint, _vp]),
    "mb200_resize_copy_channels_dev": (_i, [_vp, _sz, _sz, _i, _vp, _sz, _sz, _i, C.c_uint, _vp]),
    "mb200_restore_channels": (_i, [_vp, _vp, _sz, _sz, _i, C.c_uint]),
    "mb200_resize_copy_channels": (_i, [_vp, _sz, _sz, _i, _vp, _sz, _sz, _i, C.c_uint]),
    "mb200_statistic_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _i, _sz, _sz, _vp]),
    "mb200_rotational_blur_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _d, _vp]),
    "mb200_bilateral_blur_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _sz, _sz, _d, _d, _vp]),
    "mb200_adaptive_blur_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d, _vp]),
    "mb200_adaptive_sharpen_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d, _vp]),
    "mb200_adaptive_blur_image": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d]),
    "mb200_adaptive_sharpen_image": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d]),
    "mb200_selective_blur_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d, _d, _vp]),
    "mb200_selective_blur_image": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d, _d]),
    "mb200_statistic_image": (_i, [_vp, _vp, _sz, _sz, _i, _i, _sz, _sz]),
    "mb200_rotational_blur_image": (_i, [_vp, _vp, _sz, _sz, _i, _d]),
    "mb200_bilateral_blur_image": (_i, [_vp, _vp, _sz, _sz, _i, _sz, _sz, _d, _d]),
    "mb200_despeckle_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _vp]),
    "mb200_local_contrast_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d, _vp]),
    "mb200_wavelet_denoise_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d, _vp]),
    "mb200_despeckle_image": (_i, [_vp, _vp, _sz, _sz, _i]),
    "mb200_local_contrast_image": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d]),
    "mb200_wavelet_denoise_image": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d]),
    "mb200_emboss_kernel": (KernelPtr, [_d, _d]),
    "mb200_equalize_image_dev": (_i, [_vp, _sz, _sz, _i, _i, _vp]),
    "mb200_emboss_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d, _vp]),
    "mb200_equalize_image": (_i, [_vp, _sz, _sz, _i, _i]),
    "mb200_emboss_image": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d]),
    "mb200_sharpen_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d, _vp]),
    "mb200_edge_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _d, _vp]),
    "mb200_sharpen_image": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d]),
    "mb200_edge_image": (_i, [_vp, _vp, _sz, _sz, _i, _d]),
    "mb200_sample_image_dev": (_i, [_vp, _sz, _sz, _i, _vp, _sz, _sz, _vp]),
    "mb200_sample_image": (_i, [_vp, _sz, _sz, _i, _vp, _sz, _sz]),
    "mb200_scale_image_dev": (_i, [_vp, _sz, _sz, _i, _vp, _sz, _sz, _vp]),
    "mb200_scale_image": (_i, [_vp, _sz, _sz, _i, _vp, _sz, _sz]),
    "mb200_scale_contributions": (_l, [_i, _sz, _sz, C.POINTER(_l), C.POINTER(_i), C.POINTER(_d), _sz]),
    "mb200_thumbnail_image_dev": (_i, [_vp, _sz, _sz, _i, _vp, _sz, _sz, _i, _vp]),
    "mb200_thumbnail_image": (_i, [_vp, _sz, _sz, _i, _vp, _sz, _sz, _i]),
    "mb200_motion_blur_kernel": (_l, [_d, _d, _d, C.POINTER(_d), C.POINTER(_l), C.POINTER(_l), _sz]),
    "mb200_motion_blur_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d, _d, _vp]),
    "mb200_motion_blur_image": (_i, [_vp, _vp, _sz, _sz, _i, _d, _d, _d]),
    "mb200_bilevel_image_dev": (_i, [_vp, _sz, _sz, _i, _d, _vp]),
    "mb200_black_threshold_image_dev": (_i, [_vp, _sz, _sz, _i, _i, C.c_char_p, _vp]),
    "mb200_white_threshold_image_dev": (_i, [_vp, _sz, _sz, _i, _i, C.c_char_p, _vp]),
    "mb200_clamp_image_dev": (_i, [_vp, _sz, _sz, _i, _vp]),
    "mb200_bilevel_image": (_i, [_vp, _sz, _sz, _i, _d]),
    "mb200_black_threshold_image": (_i, [_vp, _sz, _sz, _i, _i, C.c_char_p]),
    "mb200_white_threshold_image": (_i, [_vp, _sz, _sz, _i, _i, C.c_char_p]),
    "mb200_clamp_image": (_i, [_vp, _sz, _sz, _i]),
    "mb200_adaptive_threshold_image_dev": (_i, [_vp, _vp, _sz, _sz, _i, _sz, _sz, _d, C.c_uint, _vp]),
    "mb200_auto_threshold_image_dev": (_i, [_vp, _sz, _sz, _i, _i, C.POINTER(_d), _vp]),
    "mb200_range_threshold_image_dev": (_i, [_vp, _sz, _sz, _i, _d, _d, _d, _d, _i, C.c_uint, _vp]),
    "mb200_perceptible_image_dev": (_i, [_vp, _sz, _sz, _i, _d, C.c_uint, _vp]),
    "mb200_adaptive_threshold_image": (_i, [_vp, _vp, _sz, _sz, _i, _sz, _sz, _d, C.c_uint]),
    "mb200_auto_threshold_image": (_i, [_vp, _sz, _sz, _i, _i, C.POINTER(_d)]),
    "mb200_range_threshold_image": (_i, [_vp, _sz, _sz, _i, _d, _d, _d, _d, _i, C.c_uint]),
    "mb200_perceptible_image": (_i, [_vp, _sz, _sz, _i, _d, C.c_uint]),
    "mb200_contrast_image_dev": (_i, [_vp, _sz, _sz, _i, _i, _vp]),
    "mb200_modulate_image_dev": (_i, [_vp, _sz, _sz, _i, _d, _d, _d, _i, _i, _vp]),
    "mb200_grayscale_image_dev": (_i, [_vp, _sz, _sz, _i, _i, _i, _vp]),
    "mb200_function_image_dev": (_i, [_vp, _sz, _sz, _i, _i, _sz, C.POINTER(_d), C.c_uint, _vp]),
    "mb200_contrast_image": (_i, [_vp, _sz, _sz, _i, _i]),
    "mb200_modulate_image": (_i, [_vp, _sz, _sz, _i, _d, _d, _d, _i, _i]),
    "mb200_grayscale_image": (_i, [_vp, _sz, _sz, _i, _i, _i]),
    "mb200_function_image": (_i, [_vp, _sz, _sz, _i, _i, _sz, C.POINTER(_d), C.c_uint]),
    "mb200_contrast_stretch_image_dev": (_i, [_vp, _sz, _sz, _i, _d, _d, _i, C.c_uint, _vp, _vp, _vp]),
    "mb200_contrast_stretch_image": (_i, [_vp, _sz, _sz, _i, _d, _d, _i, C.c_uint, _vp, _vp]),
    "mb200_linear_stretch_image_dev": (_i, [_vp, _sz, _sz, _i, _d, _d, C.c_uint, _vp, _vp, _vp]),
    "mb200_linear_stretch_image": (_i, [_vp, _sz, _sz, _i, _d, _d, C.c_uint, _vp, _vp]),
    "mb200_level_image_dev": (_i, [_vp, _sz, _sz, _i, _d, _d, _d, C.c_uint, _vp]),
    "mb200_level_image": (_i, [_vp, _sz, _sz, _i, _d, _d, _d, C.c_uint]),
    "mb200_levelize_image_dev": (_i, [_vp, _sz, _sz, _i, _d, _d, _d, C.c_uint, _vp]),
    "mb200_levelize_image": (_i, [_vp, _sz, _sz, _i, _d, _d, _d, C.c_uint]),
    "mb200_minmax_stretch_image_dev": (_i, [_vp, _sz, _sz, _i, _d, _d, _d, _i, C.c_uint, _vp]),
    "mb200_minmax_stretch_image": (_i, [_vp, _sz, _sz, _i, _d, _d, _d, _i, C.c_uint]),
    "mb200_gamma_image_dev": (_i, [_vp, _sz, _sz, _i, _d, C.c_uint, _vp]),
    "mb200_gamma_image": (_i, [_vp, _sz, _sz, _i, _d, C.c_uint]),
    "mb200_identify_gray_dev": (_i, [_vp, _sz, _sz, _i, _vp, _vp]),
    "mb200_identify_gray": (_i, [_vp, _sz, _sz, _i, _vp]),
}

_lib = None


def load() -> C.CDLL:
    """Loads the shared library (once) and installs the prototypes."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise RuntimeError(
            f"{LIB_PATH} is missing: the CUDA library has not been built "
            "(run `python -m imagemagick_b200.build`); there is no CPU fallback")
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)          # AttributeError == symbol not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != OK:
        msg = load().mb200_last_error()
        raise MagickB200Error(rc, msg.decode("utf-8", "replace") if msg else "")
