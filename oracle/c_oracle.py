"""ctypes binding of oracle/lexp_oracle.c (TEST / BASELINE INFRASTRUCTURE ONLY)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liblexp_oracle.so")


def build(force=False):
    src = os.path.join(_HERE, "lexp_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s", "-B", "liblexp_oracle.so"])
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            build()
        L = C.CDLL(_SO)
        L.oracle_create.restype = C.c_void_p
        L.oracle_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_float, C.c_float, C.c_float]
        L.oracle_destroy.argtypes = [C.c_void_p]
        L.oracle_set_volume.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.oracle_set_image.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.oracle_get_stats.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.oracle_sample.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.oracle_unary.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.oracle_unary_batch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_int, C.c_int]
        L.oracle_filter_unary_batch.restype = C.c_int
        L.oracle_filter_unary_batch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_int, C.c_int, C.c_int, C.c_double]
        L.oracle_max_threads.restype = C.c_int
        L.oracle_grid_mincut.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_double)]
        _lib = L
    return _lib


class COracle:
    def __init__(self, H, W, D, windR, eps, th_col, max_disp, min_disp=0.0):
        self.H, self.W, self.D = H, W, D
        self._h = lib().oracle_create(H, W, D, windR, eps, th_col, min_disp, max_disp)
        self._keep = {}
        self._guide = set()

    def close(self):
        if self._h:
            lib().oracle_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_image(self, mode, bgr):
        bgr = np.ascontiguousarray(bgr, dtype=np.uint8)
        assert bgr.shape == (self.H, self.W, 3)
        lib().oracle_set_image(self._h, mode, bgr.ctypes.data)
        self._guide.add(mode)

    def set_volume(self, mode, vol):
        vol = np.ascontiguousarray(vol, dtype=np.float32)
        assert vol.shape == (self.D, self.H, self.W)
        self._keep[mode] = vol
        lib().oracle_set_volume(self._h, mode, vol.ctypes.data)

    def stats(self, mode):
        out = np.empty((9, self.H, self.W), dtype=np.float32)
        lib().oracle_get_stats(self._h, mode, out.ctypes.data)
        return out

    def sample(self, mode, frect, plane):
        fx, fy, fw, fh = frect
        raw = np.empty((fh, fw), dtype=np.float32)
        pl = np.ascontiguousarray(plane, dtype=np.float32)
        lib().oracle_sample(self._h, mode, fx, fy, fw, fh, pl.ctypes.data, raw.ctypes.data)
        return raw

    def unary(self, mode, frect, trect, plane, with_check=True):
        fr = np.asarray(frect, dtype=np.int32)
        tr = np.asarray(trect, dtype=np.int32)
        pl = np.ascontiguousarray(plane, dtype=np.float32)
        out = np.empty((tr[3], tr[2]), dtype=np.float32)
        lib().oracle_unary(self._h, mode, fr.ctypes.data, tr.ctypes.data, pl.ctypes.data, out.ctypes.data, int(tr[2]),
                           int(with_check))
        return out

    def unary_batch(self, mode, frects, trects, planes, out_image, with_check=True, nthreads=0):
        fr = np.ascontiguousarray(frects, dtype=np.int32)
        tr = np.ascontiguousarray(trects, dtype=np.int32)
        pl = np.ascontiguousarray(planes, dtype=np.float32)
        assert out_image.dtype == np.float32 and out_image.shape == (self.H, self.W) and out_image.flags.c_contiguous
        lib().oracle_unary_batch(self._h, mode, len(fr), fr.ctypes.data, tr.ctypes.data, pl.ctypes.data,
                                 out_image.ctypes.data, int(with_check), int(nthreads))
        return out_image

    FILTER_BILATERAL, FILTER_NONE = 1, 2   # LEXP_FILTER_BILATERAL, LEXP_FILTER_NONE

    def filter_unary_batch(self, mode, frects, trects, planes, out_q=None, out_scale=None, with_check=True, filter=FILTER_BILATERAL,
                           windR=None, sig2=10.0):
        """The bilateral filter ("BL", radius windR, sig2 as the reference's float filter_param1) or none ("") of the cost-volume
        energy on every call's targetRect: (q, sum w |p|) as float64 [H][W] images, written on the targetRects only."""
        fr = np.ascontiguousarray(frects, dtype=np.int32).reshape(-1, 4)
        tr = np.ascontiguousarray(trects, dtype=np.int32).reshape(-1, 4)
        pl = np.ascontiguousarray(planes, dtype=np.float32).reshape(-1, 4)
        assert len(fr) == len(tr) == len(pl) and mode in self._keep
        if filter == self.FILTER_BILATERAL:
            assert mode in self._guide and windR is not None
        if out_q is None:
            out_q = np.full((self.H, self.W), np.nan)
        if out_scale is None:
            out_scale = np.full((self.H, self.W), np.nan)
        for a in (out_q, out_scale):
            assert a.dtype == np.float64 and a.shape == (self.H, self.W) and a.flags.c_contiguous
        if lib().oracle_filter_unary_batch(self._h, mode, len(fr), fr.ctypes.data, tr.ctypes.data, pl.ctypes.data, out_q.ctypes.data,
                                           out_scale.ctypes.data, int(with_check), int(filter), int(windR or 0),
                                           float(np.float32(sig2))):
            raise ValueError(f"oracle_filter_unary_batch: filter {filter}, sig2 {sig2}")
        return out_q, out_scale


def max_threads():
    return lib().oracle_max_threads()


def grid_mincut(tr, cap):
    """Minimum cut of an expansion-move graph: tr float32 [h][w] net terminal capacities (source - sink), cap float32 [4][h][w]
    forward arc capacities (GE, EG, LG, GG).  Returns (mask bool [h][w]: True = SOURCE segment = takes the proposal, max flow)."""
    tr = np.ascontiguousarray(tr, dtype=np.float32)
    cap = np.ascontiguousarray(cap, dtype=np.float32)
    h, w = tr.shape
    assert cap.shape == (4, h, w)
    mask = np.empty((h, w), np.uint8)
    f = C.c_double(0.0)
    if lib().oracle_grid_mincut(w, h, tr.ctypes.data, cap.ctypes.data, mask.ctypes.data, C.byref(f)):
        raise MemoryError("oracle_grid_mincut")
    return mask.astype(bool), f.value
