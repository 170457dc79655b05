"""TEST INFRASTRUCTURE ONLY.  ctypes binding of oracle/_ref/liblexp_ref_vis.so (oracle/build_ref_vis.py): the images the reference's own
Evaluator::evaluate and viewConsistencyCheck write for a given state, captured at cv::imwrite."""
import ctypes as C
import tempfile

import numpy as np

from oracle import build_ref_vis

_lib = None


def available():
    return build_ref_vis.available()


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build_ref_vis.LIB)
        P = C.c_void_p
        L.ref_vis_last_error.restype = C.c_char_p
        L.ref_vis_evaluate.argtypes = [C.c_int, C.c_int, P, P, C.c_float, P, P, P, C.c_float, C.c_float, C.c_int, C.c_char_p, P, P, P]
        L.ref_vis_check.argtypes = [C.c_int, C.c_int, P, P, C.c_float, C.c_float, P, P, P, P]
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise RuntimeError("reference image library: " + lib().ref_vis_last_error().decode())


def _c(a, dt):
    return np.ascontiguousarray(a, dtype=dt)


def evaluate_images(imL, imR, max_disp, labeling, gt, nonocc, precision, threshold, mode=0):
    """The reference's Evaluator::evaluate of view `mode` with saving on: (D, N, E) as imwrite receives them -- float32 [H][W] and
    [H][W][3] (BGR) before imwrite's 8-bit conversion, uint8 [H][W]."""
    imL, imR = _c(imL, np.uint8), _c(imR, np.uint8)
    H, W = imL.shape[:2]
    lab, g, m = _c(labeling, np.float32), _c(gt, np.float32), _c(nonocc, np.uint8)
    d, n, e = np.zeros((H, W), np.float32), np.zeros((H, W, 3), np.float32), np.zeros((H, W), np.uint8)
    with tempfile.TemporaryDirectory() as tmp:
        _check(lib().ref_vis_evaluate(H, W, imL.ctypes.data, imR.ctypes.data, float(max_disp), lab.ctypes.data, g.ctypes.data, m.ctypes.data,
                                      float(precision), float(threshold), int(mode), (tmp + "/").encode(), d.ctypes.data, n.ctypes.data,
                                      e.ctypes.data))
    return d, n, e


def check_images(imL, imR, min_disp, max_disp, lab0, lab1):
    """The reference's viewConsistencyCheck of the two labelings: (C0, C1), uint8 [H][W][3] (BGR)."""
    imL, imR = _c(imL, np.uint8), _c(imR, np.uint8)
    H, W = imL.shape[:2]
    a, b = _c(lab0, np.float32), _c(lab1, np.float32)
    c0, c1 = np.zeros((H, W, 3), np.uint8), np.zeros((H, W, 3), np.uint8)
    _check(lib().ref_vis_check(H, W, imL.ctypes.data, imR.ctypes.data, float(min_disp), float(max_disp), a.ctypes.data, b.ctypes.data,
                               c0.ctypes.data, c1.ctypes.data))
    return c0, c1
