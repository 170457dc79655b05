"""TEST INFRASTRUCTURE ONLY.  ctypes binding of oracle/_ref/liblexp_ref_run.so (oracle/build_ref_run.py): the reference's own random start
of initCurrentFast, its real Evaluator::evaluate, and its whole MidV2 run."""
import ctypes as C
import os
import tempfile

import numpy as np

from oracle import build_ref_run

_lib = None


def available():
    return build_ref_run.available()


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_ref_run.LIB)
        P = C.c_void_p
        L.ref_run_last_error.restype = C.c_char_p
        L.ref_run_random_start.argtypes = [C.c_int, C.c_int, P, P, C.c_float, C.c_int, P, P, P]
        L.ref_run_evaluate.argtypes = [C.c_int, C.c_int, P, P, C.c_float, P, P, P, P, C.c_float, C.c_float, C.c_char_p, P]
        L.ref_run_midv2.argtypes = [C.c_int, C.c_int, P, P, P, P, C.c_int, C.c_float, C.c_int, C.c_float, C.c_int, C.c_int, C.c_int,
                                    C.c_uint, C.c_char_p, P]
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise RuntimeError("reference run library: " + lib().ref_run_last_error().decode())


def _c(a, dt):
    return np.ascontiguousarray(a, dtype=dt)


def random_start(imL, imR, max_disp, units, states):
    """selectRandomPixelInRect + createRandomLabel of the reference for every unit, cv::theRNG().state = states[i] before unit i."""
    imL, imR = _c(imL, np.uint8), _c(imR, np.uint8)
    u = _c(units, np.int32).reshape(-1, 4)
    st = _c(states, np.uint64)
    out = np.zeros((len(u), 4), np.float32)
    _check(lib().ref_run_random_start(imL.shape[0], imL.shape[1], imL.ctypes.data, imR.ctypes.data, float(max_disp), len(u), u.ctypes.data,
                                      st.ctypes.data, out.ctypes.data))
    return out


def evaluate(imL, imR, max_disp, labeling, cost, gt, nonocc, precision, threshold):
    """The reference's Evaluator::evaluate of view 0: dict of valid_pixels, nonocc_pixels, all (lastAccuracy, full precision) and the log
    line's fields (log_all / log_nonocc / log_energy / log_data / log_smooth as the file has them, `%lf`)."""
    imL, imR = _c(imL, np.uint8), _c(imR, np.uint8)
    H, W = imL.shape[:2]
    lab, cst, g, m = _c(labeling, np.float32), _c(cost, np.float32), _c(gt, np.float32), _c(nonocc, np.uint8)
    out = np.zeros(9, np.float64)
    with tempfile.TemporaryDirectory() as d:
        _check(lib().ref_run_evaluate(H, W, imL.ctypes.data, imR.ctypes.data, float(max_disp), lab.ctypes.data, cst.ctypes.data, g.ctypes.data,
                                      m.ctypes.data, float(precision), float(threshold), (d + "/").encode(), out.ctypes.data))
    return dict(valid_pixels=int(out[0]), nonocc_pixels=int(out[1]), all=float(out[2]), log_energy=out[4], log_data=out[5],
                log_smooth=out[6], log_all=out[7], log_nonocc=out[8])


def midv2(imL, imR, gt, nonocc, ndisp, gt_prec, seed, iterations=5, pm_iterations=2, do_dual=True, windR=20, lam=1.0):
    """main.cpp's MidV2 with the reference's FastGCStereo::run and Evaluator: the last log line of view 0 as a dict."""
    imL, imR = _c(imL, np.uint8), _c(imR, np.uint8)
    H, W = imL.shape[:2]
    g, m = _c(gt, np.float32), _c(nonocc, np.uint8)
    out = np.zeros(6, np.float64)
    with tempfile.TemporaryDirectory() as d:
        _check(lib().ref_run_midv2(H, W, imL.ctypes.data, imR.ctypes.data, g.ctypes.data, m.ctypes.data, int(ndisp), float(gt_prec), int(windR),
                                   float(lam), int(iterations), int(pm_iterations), int(do_dual), int(seed), (d + "/").encode(),
                                   out.ctypes.data))
    return dict(time=out[0], energy=out[1], data=out[2], smooth=out[3], all=out[4], nonocc=out[5])
