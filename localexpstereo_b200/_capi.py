"""ctypes binding of the C-ABI in include/lexp_cuda.h (localexpstereo_b200/liblexp_cuda.so).

There is no fallback: if the shared library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "liblexp_cuda.so")


class LexpError(RuntimeError):
    pass


class Rect(C.Structure):  # cv::Rect
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("width", C.c_int), ("height", C.c_int)]


class PlaneC(C.Structure):  # Plane.h:4-8
    _fields_ = [("a", C.c_float), ("b", C.c_float), ("c", C.c_float), ("v", C.c_float)]


class Params(C.Structure):
    _fields_ = [("height", C.c_int), ("width", C.c_int), ("ndisp", C.c_int), ("windR", C.c_int), ("eps", C.c_float),
                ("th_col", C.c_float), ("min_disp", C.c_float), ("max_disp", C.c_float), ("device", C.c_int),
                ("energy_kind", C.c_int), ("alpha", C.c_float), ("th_grad", C.c_float), ("filter", C.c_int),
                ("reserved", C.c_int * 3)]


FILTER_GF, FILTER_BILATERAL, FILTER_NONE = 0, 1, 2   # LEXP_FILTER_* of include/lexp_cuda.h


class EvalResult(C.Structure):  # lexp_eval_result
    _fields_ = [("energy", C.c_double), ("data", C.c_double), ("smooth", C.c_double), ("valid_pixels", C.c_int64),
                ("nonocc_pixels", C.c_int64), ("all_correct", C.c_int64), ("nonocc_correct", C.c_int64), ("all", C.c_double),
                ("nonocc", C.c_double)]


class RunOptions(C.Structure):  # lexp_run_options
    _fields_ = [("n_views", C.c_int), ("pm_iterations", C.c_int), ("iterations", C.c_int), ("n_layers", C.c_int),
                ("unit_sizes", C.c_void_p), ("n_proposers", C.c_void_p), ("proposer_kind", C.c_void_p), ("proposer_K", C.c_void_p),
                ("init_labeling", C.c_void_p), ("seed", C.c_uint64), ("precision", C.c_float), ("threshold", C.c_float)]


# lexp_run_callback(user, index, mode, result, seconds)
RUN_CALLBACK = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_int, C.POINTER(EvalResult), C.c_double)
# lexp_run_image_callback(user, index, mode, kind, pixels, width, height, channels)
RUN_IMAGE_CALLBACK = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int)
IMAGE_KINDS = "DNEC"   # LEXP_IMAGE_D, _N, _E, _C of include/lexp_cuda.h

# every symbol include/lexp_cuda.h declares: (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    "lexp_last_error": (C.c_char_p, []),
    "lexp_version": (C.c_int, []),
    "lexp_create": (C.c_int, [C.POINTER(Params), C.POINTER(_P)]),
    "lexp_destroy": (C.c_int, [_P]),
    "lexp_set_image": (C.c_int, [_P, C.c_int, _P, C.c_ssize_t]),
    "lexp_set_volume_host": (C.c_int, [_P, C.c_int, _P]),
    "lexp_set_volume_device": (C.c_int, [_P, C.c_int, _P]),
    "lexp_set_volume_host_ex": (C.c_int, [_P, C.c_int, _P, C.c_int]),
    "lexp_set_volume_device_ex": (C.c_int, [_P, C.c_int, _P, C.c_int]),
    "lexp_get_stats": (C.c_int, [_P, C.c_int, _P]),
    "lexp_eval_cell": (C.c_int, [_P, C.c_int, C.POINTER(Rect), C.POINTER(Rect), C.POINTER(PlaneC), _P, C.c_ssize_t, C.c_int]),
    "lexp_eval_batch": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P, _P, C.c_ssize_t, C.c_int]),
    "lexp_plan_create": (C.c_int, [_P, C.c_int, _P, _P, C.POINTER(_P)]),
    "lexp_plan_destroy": (C.c_int, [_P]),
    "lexp_plan_num_calls": (C.c_int, [_P]),
    "lexp_plan_num_items": (C.c_int, [_P]),
    "lexp_plan_work": (C.c_int, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "lexp_plan_eval_device": (C.c_int, [_P, _P, C.c_int, _P, C.c_int, _P, C.c_ssize_t, C.c_int]),
    "lexp_plan_eval_device_tiles": (C.c_int, [_P, _P, C.c_int, _P, C.c_int, _P, C.c_int]),
    "lexp_plan_eval_host": (C.c_int, [_P, _P, C.c_int, _P, _P, C.c_ssize_t, C.c_int]),
    "lexp_plan_eval_host_tiles": (C.c_int, [_P, _P, C.c_int, _P, _P, C.c_int]),
    "lexp_host_register": (C.c_int, [_P, C.c_size_t]),
    "lexp_host_unregister": (C.c_int, [_P]),
    "lexp_sync": (C.c_int, [_P]),
    "lexp_stream": (_P, [_P]),
    "lexp_set_stream": (C.c_int, [_P, _P]),
    "lexp_set_overlap": (C.c_int, [_P, C.c_int]),
    "lexp_launch_count": (C.c_int64, [_P]),
    "lexp_overlapped_launch_count": (C.c_int64, [_P]),
    "lexp_lean_launch_count": (C.c_int64, [_P]),
    "lexp_combine_stats": (C.c_int, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "lexp_pm_begin": (C.c_int, [_P, C.c_int, _P, _P]),
    "lexp_pm_get": (C.c_int, [_P, C.c_int, _P, _P]),
    "lexp_pm_device_state": (C.c_int, [_P, C.c_int, C.POINTER(_P), C.POINTER(_P)]),
    "lexp_plan_set_units": (C.c_int, [_P, _P, _P]),
    "lexp_plan_pm_step": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint64, _P, C.c_int, _P, C.c_int]),
    "lexp_plan_pm_step_ex": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint64, _P, C.c_int, _P, C.c_int, C.c_int, _P, C.c_uint]),
    "lexp_pm_reset_sync": (C.c_int, [_P]),
    "lexp_pm_advance_epoch": (C.c_int, [_P, C.c_int, C.c_int]),
    "lexp_pm_ipc_export": (C.c_int, [_P, C.c_int, _P]),
    "lexp_pm_ipc_connect": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P]),
    "lexp_pm_connect_local": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P]),
    "lexp_pm_sweep_create": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P, _P, C.c_int, C.c_int, C.POINTER(_P)]),
    "lexp_pm_sweep_destroy": (C.c_int, [_P]),
    "lexp_pm_sweep_num_init_labels": (C.c_int, [_P]),
    "lexp_pm_sweep_init": (C.c_int, [_P, _P]),
    "lexp_pm_sweep_iteration": (C.c_int, [_P, C.c_int, C.c_uint64, C.POINTER(C.c_int)]),
    "lexp_pm_sweep_gc_iteration": (C.c_int, [_P, C.c_int, C.c_uint64, C.POINTER(C.c_int)]),
    "lexp_set_smoothness": (C.c_int, [_P, C.c_float, C.c_float, C.c_float, C.c_float]),
    "lexp_get_smooth_coeff": (C.c_int, [_P, C.c_int, _P]),
    "lexp_pairwise_terms": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P]),
    "lexp_plan_init_step": (C.c_int, [_P, _P, C.c_int, _P, C.c_int]),
    "lexp_pm_init_from_labeling": (C.c_int, [_P, C.c_int]),
    "lexp_set_volume_file": (C.c_int, [_P, C.c_int, C.c_char_p, C.c_int]),
    "lexp_get_disparities": (C.c_int, [_P, C.c_int, _P]),
    "lexp_save_pfm": (C.c_int, [C.c_char_p, _P, C.c_int, C.c_int, C.c_ssize_t]),
    "lexp_post_process": (C.c_int, [_P, C.c_float, _P]),
    "lexp_energy": (C.c_int, [_P, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "lexp_plan_gc_step": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_uint64, _P, C.c_int, _P, _P]),
    "lexp_pm_sweep_init_random": (C.c_int, [_P, C.c_uint64]),
    "lexp_set_ground_truth": (C.c_int, [_P, _P, _P]),
    "lexp_evaluate": (C.c_int, [_P, C.c_int, C.c_float, C.c_float, C.POINTER(EvalResult)]),
    "lexp_run_seed": (C.c_uint64, [C.c_uint64, C.c_int, C.c_int, C.c_int]),
    "lexp_run": (C.c_int, [_P, C.POINTER(RunOptions), _P, _P, RUN_CALLBACK, _P]),
    "lexp_render_evaluation": (C.c_int, [_P, C.c_int, C.c_float, C.c_float, _P, _P, _P]),
    "lexp_render_consistency": (C.c_int, [_P, _P, _P]),
    "lexp_run_ex": (C.c_int, [_P, C.POINTER(RunOptions), _P, _P, RUN_CALLBACK, RUN_IMAGE_CALLBACK, _P]),
    "lexp_layer_geometry": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), _P, _P, _P, _P]),
}

_lib = None


def lib():
    """Loads liblexp_cuda.so (once).  Raises LexpError if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise LexpError(f"{SO_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                            "(there is no CPU fallback)")
        L = C.CDLL(SO_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)  # AttributeError if the library does not export it
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        raise LexpError(f"lexp error {rc}: {lib().lexp_last_error().decode()}")
