"""TEST INFRASTRUCTURE ONLY.  ctypes binding of oracle/_ref/liblexp_ref_filters.so (oracle/ref_filter_driver.cpp): the reference's own
CostVolumeEnergy ("BL" / "") and NaiveStereoEnergy ("BF" / "") with their BilateralFilter, compiled from its headers."""
import ctypes as C
import os

import numpy as np

from oracle import build_ref_filters as B

_lib = None


def available():
    return B.available()


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(B.LIB)
        P = C.c_void_p
        L.ref_filter_last_error.restype = C.c_char_p
        L.ref_filter_create.restype = P
        L.ref_filter_create.argtypes = [C.c_int] * 4 + [P] * 4 + [C.c_int, C.c_char_p] + [C.c_float] * 6
        L.ref_filter_destroy.argtypes = [P]
        L.ref_filter_unary.restype = C.c_int
        L.ref_filter_unary.argtypes = [P, P, P, P, C.c_int, C.c_int, P]
        _lib = L
    return _lib


class RefFilterEnergy:
    """kind 0: CostVolumeEnergy(imL, imR, volL, volR, Parameters(windR, filter_name, param1), MAX, MIN); kind 1: NaiveStereoEnergy."""

    def __init__(self, kind, imL, imR, volL, volR, windR, filter_name, param1, th_col, th_grad, alpha, max_disp, min_disp=0.0):
        H, W = imL.shape[:2]
        self.keep = [np.ascontiguousarray(imL, np.uint8), np.ascontiguousarray(imR if imR is not None else imL, np.uint8)]
        D = 1
        vols = [None, None]
        if kind == 0:
            D = volL.shape[0]
            vols = [np.ascontiguousarray(volL, np.float32), np.ascontiguousarray(volR if volR is not None else volL, np.float32)]
            self.keep += vols
        self.h = lib().ref_filter_create(kind, H, W, D, self.keep[0].ctypes.data, self.keep[1].ctypes.data,
                                         vols[0].ctypes.data if kind == 0 else None, vols[1].ctypes.data if kind == 0 else None,
                                         int(windR), filter_name.encode(), float(param1), float(th_col), float(th_grad), float(alpha),
                                         float(max_disp), float(min_disp))
        if not self.h:
            raise RuntimeError(lib().ref_filter_last_error().decode())

    def unary(self, frect, trect, plane, mode=0, with_check=True):
        """costs(targetRect) as the reference writes them, float32 [th][tw]."""
        fx, fy, fw, fh = (int(v) for v in frect)
        tx, ty, tw, th = (int(v) for v in trect)
        out = np.full((fh, fw), np.float32(-7.0), np.float32)
        fr = np.array([fx, fy, fw, fh], np.int32)
        tr = np.array([tx, ty, tw, th], np.int32)
        pl = np.ascontiguousarray(plane, np.float32)
        if lib().ref_filter_unary(self.h, fr.ctypes.data, tr.ctypes.data, pl.ctypes.data, int(mode), int(bool(with_check)), out.ctypes.data):
            raise RuntimeError(lib().ref_filter_last_error().decode())
        return out[ty - fy:ty - fy + th, tx - fx:tx - fx + tw].copy()

    def close(self):
        if self.h:
            lib().ref_filter_destroy(self.h)
            self.h = None
