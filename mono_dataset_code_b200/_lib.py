"""ctypes binding of libmdc_b200.so (the C ABI declared in include/mdc_b200.h).

There is no CPU fallback: if the shared library is missing this module raises at import
time, and every per-frame call goes into the sm_90a kernels.
"""
from __future__ import annotations

import ctypes as C
import os

PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG, "lib", "libmdc_b200.so")

MDC_OK = 0
ERR_NAMES = {1: "INVALID_ARG", 2: "IO", 3: "FORMAT", 4: "INVALID_OBJECT", 5: "CUDA", 6: "UNSUPPORTED"}
RECTIFY, REMOVE_GAMMA, REMOVE_VIGNETTE, NAN_OVEREXPOSED = 1, 2, 4, 8
FOV_CROP, FOV_FULL, FOV_EXPLICIT = -1, -2, 0
MAX_PYR_LEVELS = 8

_f32p = C.POINTER(C.c_float)
_vp = C.c_void_p

# every exported symbol of include/mdc_b200.h: name -> (restype, argtypes)
SIGNATURES = {
    "mdc_last_error": (C.c_char_p, []),
    "mdc_version": (C.c_char_p, []),
    "mdc_fov_create": (C.c_int, [C.c_char_p, C.POINTER(_vp)]),
    "mdc_fov_create_ex": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(_vp)]),
    "mdc_fov_create_from_params": (C.c_int, [_f32p, C.c_int, C.c_int, C.c_int, _f32p, C.c_int, C.c_int, C.c_int, C.POINTER(_vp)]),
    "mdc_fov_destroy": (None, [_vp]),
    "mdc_fov_is_valid": (C.c_int, [_vp]),
    "mdc_fov_dims": (C.c_int, [_vp] + [C.POINTER(C.c_int)] * 4),
    "mdc_fov_get_K": (C.c_int, [_vp, _f32p, _f32p]),
    "mdc_fov_omega": (C.c_float, [_vp]),
    "mdc_fov_original_calibration": (C.c_int, [_vp, _f32p]),
    "mdc_fov_distort_coordinates": (C.c_int, [_vp, _f32p, _f32p, C.c_int]),
    "mdc_fov_distort_coordinates_device": (C.c_int, [_vp, _vp, _vp, C.c_size_t, C.c_int, _vp]),
    "mdc_atanf_host": (None, [_f32p, _f32p, C.c_size_t]),
    "mdc_seq_open": (C.c_int, [C.c_char_p, C.POINTER(_vp)]),
    "mdc_seq_close": (None, [_vp]),
    "mdc_seq_num_images": (C.c_int, [_vp]),
    "mdc_seq_is_zipped": (C.c_int, [_vp]),
    "mdc_seq_name": (C.c_char_p, [_vp, C.c_int]),
    "mdc_seq_timestamp": (C.c_double, [_vp, C.c_int]),
    "mdc_seq_exposure": (C.c_float, [_vp, C.c_int]),
    "mdc_seq_read_gray8": (C.c_int, [_vp, C.c_int, _vp, C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "mdc_seq_prepare": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint, C.POINTER(_vp), C.c_int, C.c_int]),
    "mdc_seq_prepare_device": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_uint, C.POINTER(_vp), C.c_int, C.c_int, _vp]),
    "mdc_jpeg_decode_device": (C.c_int, [_vp, C.POINTER(_vp), C.POINTER(C.c_size_t), C.c_int, C.c_int, C.c_int, _vp, C.c_size_t,
                                         C.POINTER(C.c_int), _vp]),
    "mdc_vc_plane_step": (C.c_int, [_vp, _vp, _vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _vp, _vp, C.c_double, C.c_int, C.POINTER(C.c_double)]),
    "mdc_vc_vignette_step": (C.c_int, [_vp, _vp, _vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _vp, _vp, C.c_double, C.c_int, C.POINTER(C.c_double)]),
    "mdc_vc_smooth": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, _vp]),
    "mdc_vignette_calib": (C.c_int, [_vp, _vp, _vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp, C.POINTER(C.c_double)]),
    "mdc_vc_plane_maps": (C.c_int, [_vp, C.POINTER(C.c_double), C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, _vp, _vp, C.c_int, _vp]),
    "mdc_vc_prepare_images": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, _f32p, C.c_float, C.c_int, _vp, _vp]),
    "mdc_marker_threshold": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp]),
    "mdc_marker_detect": (C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp, C.c_int, C.POINTER(C.c_int)]),
    "mdc_marker_homography": (C.c_int, [_f32p, C.POINTER(C.c_double)]),
    "mdc_marker_contours": (C.c_int, [_vp, C.c_int, C.c_int, _vp, C.c_size_t, _vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_size_t)]),
    "mdc_marker_approx_poly": (C.c_int, [_vp, C.c_int, C.c_double, _vp, C.POINTER(C.c_int)]),
    "mdc_marker_candidates": (C.c_int, [_vp, C.c_int, C.c_int, _f32p, C.c_int, C.POINTER(C.c_int)]),
    "mdc_marker_read_patch": (C.c_int, [_vp, C.c_int, C.c_int, _f32p, _vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "mdc_atanf_device": (C.c_int, [_vp, _vp, C.c_size_t, C.c_int, _vp]),
    "mdc_fov_remap_x": (_f32p, [_vp]),
    "mdc_fov_remap_y": (_f32p, [_vp]),
    "mdc_photo_create": (C.c_int, [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.POINTER(_vp)]),
    "mdc_photo_create_from_arrays": (C.c_int, [_f32p, _vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_vp)]),
    "mdc_photo_destroy": (None, [_vp]),
    "mdc_photo_valid_gamma": (C.c_int, [_vp]),
    "mdc_photo_valid_vignette": (C.c_int, [_vp]),
    "mdc_photo_ginv": (_f32p, [_vp]),
    "mdc_photo_g": (_f32p, [_vp]),
    "mdc_photo_vignette_map": (_f32p, [_vp]),
    "mdc_photo_vignette_map_inv": (_f32p, [_vp]),
    "mdc_ctx_create": (C.c_int, [C.c_int, _vp, _vp, C.POINTER(_vp)]),
    "mdc_ctx_create_from_device_tables": (C.c_int, [C.c_int] * 5 + [_vp] * 4 + [C.POINTER(_vp)]),
    "mdc_ctx_take_table_ownership": (C.c_int, [_vp]),
    "mdc_ctx_destroy": (None, [_vp]),
    "mdc_ctx_device_tables": (C.c_int, [_vp] + [C.POINTER(_vp)] * 4),
    "mdc_ctx_level_dims": (C.c_int, [_vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "mdc_ctx_launch_count": (C.c_longlong, [_vp]),
    "mdc_ctx_configure": (C.c_int, [_vp, C.c_int, C.c_int]),
    "mdc_ctx_loader_usable": (C.c_int, [_vp, C.c_int]),
    "mdc_ctx_auto_loader": (C.c_int, [_vp]),
    "mdc_ctx_loader_usable_pitched": (C.c_int, [_vp, C.c_int, C.c_size_t]),
    "mdc_ctx_auto_loader_pitched": (C.c_int, [_vp, C.c_size_t]),
    "mdc_unmap_u8": (C.c_int, [_vp, _vp, _vp, C.c_int, C.c_int, C.c_uint, _vp]),
    "mdc_undistort_u8": (C.c_int, [_vp, _vp, _vp, C.c_int, C.c_int, C.c_int, _vp]),
    "mdc_undistort_f32": (C.c_int, [_vp, _vp, _vp, C.c_int, C.c_int, C.c_int, _vp]),
    "mdc_prepare_batch": (C.c_int, [_vp, _vp, C.c_int, C.c_uint, C.POINTER(_vp), C.c_int, _vp]),
    "mdc_prepare_batch_pitched": (C.c_int, [_vp, _vp, C.c_size_t, C.c_int, C.c_uint, C.POINTER(_vp), C.c_int, _vp]),
    "mdc_pyr_down": (C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp, C.c_int, _vp]),
    "mdc_estep": (C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp, _vp, _vp, _vp]),
    "mdc_rc_leak_padding": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, _vp]),
    "mdc_rc_einit": (C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp, _vp]),
    "mdc_rc_gstep": (C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp, _vp, _vp, _vp]),
    "mdc_rc_rescale": (C.c_int, [_vp, C.c_int, _vp, _vp, C.POINTER(C.c_double)]),
    "mdc_rc_rmse": (C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp, _vp, _vp, C.POINTER(C.c_double)]),
    "mdc_response_calib": (C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp, C.c_int, _vp, _vp, C.POINTER(C.c_double)]),
    "mdc_rc_gstep_accumulate": (C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp, _vp, _vp, _vp, C.c_int, _vp]),
    "mdc_rc_gstep_finish": (C.c_int, [_vp, _vp, _vp, _vp, _vp]),
    "mdc_rc_gstep_scale": (C.c_int, [_vp, _vp, C.c_int, _vp, C.c_int, _vp, _vp]),
    "mdc_rc_gstep_accumulate_exact": (C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, C.c_int, _vp]),
    "mdc_rc_gstep_finish_exact": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mdc_rc_rmse_accumulate": (C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp]),
    "mdc_unmap_u8_host": (C.c_int, [_vp, _vp, _vp, C.c_int, C.c_uint]),
    "mdc_undistort_u8_host": (C.c_int, [_vp, _vp, _vp, C.c_int, C.c_int]),
    "mdc_undistort_f32_host": (C.c_int, [_vp, _vp, _vp, C.c_int, C.c_int]),
    "mdc_prepare_batch_host": (C.c_int, [_vp, _vp, C.c_int, C.c_uint, C.POINTER(_vp), C.c_int]),
    "mdc_host_alloc": (C.c_int, [C.POINTER(_vp), C.c_size_t]),
    "mdc_host_free": (None, [_vp]),
    "mdc_device_numa_node": (C.c_int, [C.c_int]),
}


def load() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -m mono_dataset_code_b200.build` "
            "(or __graft_entry__.build()).  There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError here = header and library out of sync
        fn.restype = res
        fn.argtypes = args
    return lib


lib = load()


class MdcError(RuntimeError):
    def __init__(self, code: int, where: str):
        self.code = code
        msg = lib.mdc_last_error().decode(errors="replace")
        super().__init__(f"{where}: MDC_ERR_{ERR_NAMES.get(code, code)}: {msg}")


def check(code: int, where: str) -> None:
    if code != MDC_OK:
        raise MdcError(code, where)
