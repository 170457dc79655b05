"""Host-side mirror of the reference's operator interface for the unary-cost path.

Same names, argument meaning and error behaviour as the reference classes
(`/root/reference/LocalExpansionStereo/`): `Plane` (Plane.h:4-106), `Parameters`
(StereoEnergy.h:13-40), `LayerManager` / `Layer` (LayerManager.h:7-186) and
`CostVolumeEnergy` with `ComputeUnaryPotential[WithoutCheck]` (StereoEnergy.h:625-626,
CostVolumeEnergy.h:55-183).  All arithmetic of the hot path runs in the CUDA library behind
the C-ABI (`include/lexp_cuda.h`); this file only marshals numpy arrays (the cv::Mat stand-in).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

from . import _capi
from ._capi import LexpError, PlaneC, Rect, check, lib

COST_FOR_INVALID = 1000000.0  # StereoEnergy.h:45


@dataclass
class Parameters:  # StereoEnergy.h:13-40 (defaults of the constructor at :26)
    lambda_: float = 20.0
    windR: int = 20
    filterName: str = "GF"
    filter_param1: float = 1e-4
    alpha: float = 0.9
    omega: float = 10.0
    th_grad: float = 2.0
    th_col: float = 10.0
    th_smooth: float = 1.0
    epsilon: float = 0.01
    neighborNum: int = 8


class Plane:
    """struct Plane {a,b,c,v} (Plane.h:4-12)."""
    __slots__ = ("a", "b", "c", "v")

    def __init__(self, a=0.0, b=0.0, c=0.0, v=0.0):
        self.a, self.b, self.c, self.v = (float(np.float32(t)) for t in (a, b, c, v))

    @staticmethod
    def CreatePlane(nx, ny, nz, z, x, y, v=0.0):  # Plane.h:14-32, float arithmetic
        f = np.float32
        nx, ny, nz, z, x, y = (f(t) for t in (nx, ny, nz, z, x, y))
        a = f(-nx / nz)
        b = f(-ny / nz)
        c = f(f(z - f(a * x)) - f(b * y))
        return Plane(a, b, c, v)

    def GetZ(self, x, y):  # Plane.h:51-54
        f = np.float32
        return float(f(f(f(f(self.a) * f(x)) + f(f(self.b) * f(y))) + f(self.c)))

    def toVec4(self):
        return np.array([self.a, self.b, self.c, self.v], dtype=np.float32)

    def __iter__(self):
        return iter((self.a, self.b, self.c, self.v))


def _as_rect(r) -> Rect:
    if isinstance(r, Rect):
        return r
    x, y, w, h = (int(t) for t in r)
    return Rect(x, y, w, h)


def _rect_array(rects) -> np.ndarray:
    a = np.ascontiguousarray(np.asarray([tuple(r) if not isinstance(r, Rect) else (r.x, r.y, r.width, r.height) for r in rects],
                                        dtype=np.int32))
    assert a.ndim == 2 and a.shape[1] == 4
    return a


def _plane_array(planes) -> np.ndarray:
    if isinstance(planes, np.ndarray):
        a = np.ascontiguousarray(planes, dtype=np.float32)
    else:
        a = np.ascontiguousarray(np.asarray([tuple(p) for p in planes], dtype=np.float32))
    assert a.ndim == 2 and a.shape[1] == 4
    return a


@dataclass
class Layer:  # LayerManager.h:14-24
    heightBlocks: int
    widthBlocks: int
    regionUnitSize: int
    unitRegions: List[tuple]
    sharedRegions: List[tuple]
    filterRegions: List[tuple]
    disjointRegionSets: List[List[int]]
    proposers: list = field(default_factory=list)


class LayerManager:
    """LayerManager (LayerManager.h:7-186); geometry computed by the C++ library (lexp_layer_geometry)."""

    def __init__(self, width, height, windowR, localLabelSetNum=0):
        self.width, self.height, self.windowR = int(width), int(height), int(windowR)
        self.layers: List[Layer] = []

    def addLayer(self, unitRegionSize):
        u = int(unitRegionSize)
        hb, wb = C.c_int(), C.c_int()
        check(lib().lexp_layer_geometry(self.width, self.height, self.windowR, u, C.byref(hb), C.byref(wb), None, None, None, None))
        n = hb.value * wb.value
        unit = np.zeros((n, 4), np.int32)
        shared = np.zeros((n, 4), np.int32)
        filt = np.zeros((n, 4), np.int32)
        grp = np.zeros(n, np.int32)
        check(lib().lexp_layer_geometry(self.width, self.height, self.windowR, u, C.byref(hb), C.byref(wb),
                                        unit.ctypes.data, shared.ctypes.data, filt.ctypes.data, grp.ctypes.data))
        sets = [[] for _ in range(16)]
        for r in range(n):
            sets[int(grp[r])].append(r)
        sets = [s for s in sets if s]  # empty groups erased (LayerManager.h:174-182)
        self.layers.append(Layer(hb.value, wb.value, u, [tuple(map(int, r)) for r in unit], [tuple(map(int, r)) for r in shared],
                                 [tuple(map(int, r)) for r in filt], sets))
        return self.layers[-1]


def host_register(array: np.ndarray):
    """Page-lock + map a numpy buffer (lexp_host_register): the host entry points then write into it zero-copy."""
    check(lib().lexp_host_register(array.ctypes.data, array.nbytes))


def save_pfm_file(path, image: np.ndarray):
    """cvutils::io::save_pfm_file (Utilities.hpp:84-137) for a 1-channel float32 image."""
    assert image.dtype == np.float32 and image.ndim == 2 and image.strides[1] == 4
    check(lib().lexp_save_pfm(str(path).encode(), image.ctypes.data, image.shape[1], image.shape[0], image.strides[0]))


def host_unregister(array: np.ndarray):
    check(lib().lexp_host_unregister(array.ctypes.data))


PROP_LIST, PROP_EXPANSION, PROP_RANDOM, PROP_RANSAC = 0, 1, 2, 3   # LEXP_PROP_* of include/lexp_cuda.h
VOL_PLAIN, VOL_FILL, VOL_RIGHT_FROM_LEFT = 0, 1, 2   # LEXP_VOL_*


class Plan:
    """Device-resident work list for a fixed list of (filterRect, targetRect) (see lexp_plan_create)."""

    def __init__(self, energy: "CostVolumeEnergy", filter_rects, target_rects):
        self.energy = energy
        self._fr = _rect_array(filter_rects)
        self._tr = _rect_array(target_rects)
        assert len(self._fr) == len(self._tr)
        h = C.c_void_p()
        check(lib().lexp_plan_create(energy._h, len(self._fr), self._fr.ctypes.data, self._tr.ctypes.data, C.byref(h)))
        self._h = h
        sf, ss, ab = C.c_int64(), C.c_int64(), C.c_int64()
        check(lib().lexp_plan_work(self._h, C.byref(sf), C.byref(ss), C.byref(ab)))
        self.filter_px, self.target_px, self.algorithmic_bytes = sf.value, ss.value, ab.value
        self.num_calls = lib().lexp_plan_num_calls(self._h)
        self.num_items = lib().lexp_plan_num_items(self._h)

    def eval_host(self, planes, cost_image: np.ndarray, with_check=True, mode=0):
        pl = _plane_array(planes)
        assert len(pl) == self.num_calls
        assert cost_image.dtype == np.float32 and cost_image.ndim == 2 and cost_image.strides[1] == 4
        check(lib().lexp_plan_eval_host(self.energy._h, self._h, mode, pl.ctypes.data, cost_image.ctypes.data,
                                        cost_image.strides[0], int(with_check)))
        return cost_image

    def eval_host_tiles(self, planes, tiles: np.ndarray, with_check=True, mode=0):
        """Per-call contiguous tiles into a host float32 array of target_px elements (tile i at sweep.tile_offsets)."""
        pl = _plane_array(planes)
        assert len(pl) == self.num_calls
        assert tiles.dtype == np.float32 and tiles.ndim == 1 and tiles.size >= self.target_px and tiles.strides[0] == 4
        check(lib().lexp_plan_eval_host_tiles(self.energy._h, self._h, mode, pl.ctypes.data, tiles.ctypes.data, int(with_check)))
        return tiles

    def _planes_ptr(self, planes, planes_on_device):
        """The planes argument of the C calls: a device pointer as given, or a host copy of num_calls planes kept alive until
        the next call (the copy out of it is asynchronous)."""
        if planes_on_device:
            return int(planes)
        self._pl_keep = _plane_array(planes)
        assert len(self._pl_keep) == self.num_calls
        return self._pl_keep.ctypes.data

    def eval_device(self, planes, d_cost_ptr: int, step_bytes: int, with_check=True, mode=0, planes_on_device=False):
        """planes: numpy [n][4] (host) or an int device pointer when planes_on_device."""
        ptr = self._planes_ptr(planes, planes_on_device)
        check(lib().lexp_plan_eval_device(self.energy._h, self._h, mode, ptr, int(planes_on_device), int(d_cost_ptr),
                                          int(step_bytes), int(with_check)))

    def eval_device_tiles(self, planes, d_tiles_ptr: int, with_check=True, mode=0, planes_on_device=False):
        """Per-call contiguous tiles at d_tiles + sum of previous targetRect areas (floats)."""
        ptr = self._planes_ptr(planes, planes_on_device)
        check(lib().lexp_plan_eval_device_tiles(self.energy._h, self._h, mode, ptr, int(planes_on_device), int(d_tiles_ptr),
                                                int(with_check)))

    # --- PatchMatch phase on the device (lexp_plan_set_units / lexp_plan_pm_step) -------------------------------------
    def set_units(self, unit_rects, cell_ids=None):
        """unitRegion of every call (LayerManager.h:117-121) and a global id per cell (seeds its random streams)."""
        u = _rect_array(unit_rects)
        assert len(u) == self.num_calls
        ids = None if cell_ids is None else np.ascontiguousarray(cell_ids, dtype=np.int32)
        check(lib().lexp_plan_set_units(self._h, u.ctypes.data, None if ids is None else ids.ctypes.data))

    def pm_step(self, step_index, kind, m=0, seed=0, planes=None, planes_on_device=False, d_planes_out=0, init=False, mode=0,
                publish_epoch=0, wait_epochs=None, wait_mask=0):
        """One proposal step of FastGCStereo.h:41-60 (doGC == false) for all cells of the plan, asynchronous:
        kind = PROP_LIST (planes: numpy [n][4] or a device pointer) | PROP_EXPANSION | PROP_RANDOM (m = outerIter + iter) |
        PROP_RANSAC (RansacProposer(1) on the state before the step; not with init)."""
        ptr = self._planes_ptr(planes, planes_on_device) if kind == PROP_LIST else None
        we = None
        if wait_mask:
            self._we_keep = np.zeros(8, np.int32)
            self._we_keep[:len(wait_epochs)] = wait_epochs
            we = self._we_keep.ctypes.data
        check(lib().lexp_plan_pm_step_ex(self.energy._h, self._h, mode, int(step_index), int(kind), int(m), int(seed) & 0xFFFFFFFFFFFFFFFF,
                                         ptr, int(planes_on_device), int(d_planes_out) or None, 1 if init else 0, int(publish_epoch), we, int(wait_mask)))

    def init_step(self, planes, planes_on_device=False, mode=0):
        """initCurrentFast (FastGCStereo.h:101-113) for any energy kind: label and unary cost of every call's targetRect, unconditionally."""
        ptr = self._planes_ptr(planes, planes_on_device)
        check(lib().lexp_plan_init_step(self.energy._h, self._h, mode, ptr, int(planes_on_device)))

    def gc_step(self, kind, m=0, seed=0, planes=None, planes_on_device=False, d_planes_out=0, d_flows_out=0, mode=0):
        """One proposal step of FastGCStereo.h:41-60 with doGC == true for all cells of the plan, asynchronous: proposal, unary cost,
        FastGCStereo::expansionMoveBK (graph of :424-549 + its minimum cut) and the copyTo / setTo of the winners -- on the device.
        d_flows_out: optional device pointer of double[n] receiving the minimum-cut energy of every move."""
        ptr = self._planes_ptr(planes, planes_on_device) if kind == PROP_LIST else None
        check(lib().lexp_plan_gc_step(self.energy._h, self._h, mode, int(kind), int(m), int(seed) & 0xFFFFFFFFFFFFFFFF, ptr,
                                      int(planes_on_device), int(d_planes_out) or None, int(d_flows_out) or None))

    def close(self):
        if self._h:
            lib().lexp_plan_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CostVolumeEnergy:
    """CostVolumeEnergy (CostVolumeEnergy.h:6-184) backed by the sm_90a kernels.

    imL / imR: uint8 [H][W][3] BGR; volL / volR: float32 [D][H][W] numpy arrays, or torch CUDA tensors /
    integer device pointers (then no copy is made).  `params.filterName`, as the reference selects the filter
    (CostVolumeEnergy.h:23-42): "GF" or "GFfloat" (both run the same FP32 guided-filter kernel, within the 1e-4 tolerance of the
    reference's double filter), "BL" (bilateral filter, sig2 = filter_param1) or "" (no filter).  Any other name is rejected: the
    reference leaves its filter a null pointer there and crashes on the first unary call."""

    ENERGY_KIND = 0
    # filterName -> LEXP_FILTER_* (include/lexp_cuda.h)
    FILTERS = {"GF": _capi.FILTER_GF, "GFfloat": _capi.FILTER_GF, "BL": _capi.FILTER_BILATERAL, "": _capi.FILTER_NONE}

    @classmethod
    def _filter_kind(cls, name):
        if name not in cls.FILTERS:
            raise LexpError(f'{cls.__name__} has no filter named "{name}": the reference leaves its filter a null pointer for that '
                            f'name and crashes in ComputeUnaryPotential; use one of {sorted(cls.FILTERS)}')
        return cls.FILTERS[name]

    def __init__(self, imL, imR, volL, volR, params: Parameters, MAX_DISPARITY, MIN_DISPARITY=0.0, MAX_VDISPARITY=0.0,
                 device: int = 0):
        filter_kind = self._filter_kind(params.filterName)
        if MAX_VDISPARITY != 0:
            raise LexpError("MAX_VDISPARITY != 0 is not supported (main.cpp never sets it)")
        imL = np.ascontiguousarray(imL, dtype=np.uint8)
        self.height, self.width = imL.shape[:2]
        self.params = params
        self.MAX_DISPARITY, self.MIN_DISPARITY = float(MAX_DISPARITY), float(MIN_DISPARITY)
        D = self._ndisp(volL) if volL is not None else int(MAX_DISPARITY) + 1
        p = _capi.Params(self.height, self.width, D, int(params.windR), float(params.filter_param1), float(params.th_col),
                         float(MIN_DISPARITY), float(MAX_DISPARITY), int(device), int(self.ENERGY_KIND), float(params.alpha),
                         float(params.th_grad), filter_kind)
        h = C.c_void_p()
        check(lib().lexp_create(C.byref(p), C.byref(h)))
        self._h = h
        self._keep = []
        self.ndisp = D
        for mode, (im, vol) in enumerate(((imL, volL), (imR, volR))):
            if im is not None:
                im = np.ascontiguousarray(im, dtype=np.uint8)
                assert im.shape == (self.height, self.width, 3)
                check(lib().lexp_set_image(self._h, mode, im.ctypes.data, im.strides[0]))
            if vol is not None:
                self._set_volume(mode, vol)

    @staticmethod
    def _ndisp(vol):
        return int(vol.shape[0])

    def _set_volume(self, mode, vol, transform=VOL_PLAIN):
        if isinstance(vol, np.ndarray):
            v = np.ascontiguousarray(vol, dtype=np.float32)
            assert v.shape == (self.ndisp, self.height, self.width)
            check(lib().lexp_set_volume_host_ex(self._h, mode, v.ctypes.data, int(transform)))
        else:  # torch CUDA tensor (duck-typed): only read during the call
            assert tuple(vol.shape) == (self.ndisp, self.height, self.width) and vol.is_contiguous() and vol.is_cuda
            check(lib().lexp_set_volume_device_ex(self._h, mode, vol.data_ptr(), int(transform)))

    def set_volume_file(self, mode, path, transform=VOL_PLAIN):
        """The reference's `.acrt` cost-volume file (raw float[D][H][W], main.cpp:353-364), streamed from disk in slabs."""
        check(lib().lexp_set_volume_file(self._h, mode, str(path).encode(), int(transform)))

    def set_volume(self, mode, vol, transform=VOL_PLAIN):
        """(Re)load the cost volume of a view with the reference's volume preparation fused into the upload (main.cpp:146-199):
        VOL_FILL = fillOutOfView(vol, mode); VOL_RIGHT_FROM_LEFT (mode 1) = the right volume derived from the LEFT one,
        fillOutOfView(convertVolumeL2R(fillOutOfView(volL, 0)), 1)."""
        self._set_volume(mode, vol, transform)

    # --- the two virtuals of StereoEnergy (StereoEnergy.h:625-626) -------------------------------
    def ComputeUnaryPotentialWithoutCheck(self, filterRect, targetRect, costs: np.ndarray, plane, reusable=None, mode=0):
        self._eval_cell(filterRect, targetRect, costs, plane, mode, 0)

    def ComputeUnaryPotential(self, filterRect, targetRect, costs: np.ndarray, plane, reusable=None, mode=0):
        self._eval_cell(filterRect, targetRect, costs, plane, mode, 1)

    def _eval_cell(self, filterRect, targetRect, costs, plane, mode, with_check):
        """`costs` is the numpy view proposalCost[fy:fy+fh, fx:fx+fw] (cv::Mat ROI at filterRect)."""
        fr, tr = _as_rect(filterRect), _as_rect(targetRect)
        assert costs.dtype == np.float32 and costs.shape == (fr.height, fr.width) and costs.strides[1] == 4
        pl = PlaneC(*[float(t) for t in plane])
        check(lib().lexp_eval_cell(self._h, mode, C.byref(fr), C.byref(tr), C.byref(pl), costs.ctypes.data, costs.strides[0],
                                   with_check))

    # --- batched forms ------------------------------------------------------------------------------
    def ComputeUnaryPotentialBatch(self, filterRects, targetRects, cost_image: np.ndarray, planes, mode=0, with_check=True):
        fr, tr, pl = _rect_array(filterRects), _rect_array(targetRects), _plane_array(planes)
        assert cost_image.dtype == np.float32 and cost_image.shape == (self.height, self.width) and cost_image.strides[1] == 4
        check(lib().lexp_eval_batch(self._h, mode, len(fr), fr.ctypes.data, tr.ctypes.data, pl.ctypes.data,
                                    cost_image.ctypes.data, cost_image.strides[0], int(with_check)))
        return cost_image

    def make_plan(self, filterRects, targetRects) -> Plan:
        return Plan(self, filterRects, targetRects)

    def stats(self, mode=0) -> np.ndarray:
        out = np.empty((9, self.height, self.width), dtype=np.float32)
        check(lib().lexp_get_stats(self._h, mode, out.ctypes.data))
        return out

    # --- pairwise terms (StereoEnergy.h:131-163, 398-453) -------------------------------------------------------------------------
    def set_smoothness(self, lam=1.0, omega=10.0, th_smooth=1.0, epsilon=0.01):
        """Parameters::lambda / omega / th_smooth / epsilon (StereoEnergy.h:26-36); the coefficient maps are rebuilt on the device."""
        check(lib().lexp_set_smoothness(self._h, float(lam), float(omega), float(th_smooth), float(epsilon)))

    def smooth_coeff(self, mode=0) -> np.ndarray:
        """smoothnessCoeff[mode] without its margin: float32 [8][H][W], neighbours in the order of StereoEnergy::NB_*."""
        out = np.empty((8, self.height, self.width), dtype=np.float32)
        check(lib().lexp_get_smooth_coeff(self._h, mode, out.ctypes.data))
        return out

    def computeSmoothnessTermsExpansion(self, regions, planes, mode=0):
        """StereoEnergy::computeSmoothnessTermsExpansion(.., onlyForward = true) for n (region, proposal) pairs on the device state of
        view `mode` (pm_begin).  Returns a list of (cost00, cost01, cost10), each float32 [4][h][w] for NB_GE, NB_EG, NB_LG, NB_GG."""
        rg, pl = _rect_array(regions), _plane_array(planes)
        assert len(rg) == len(pl)
        sizes = [int(r[2]) * int(r[3]) for r in rg.reshape(-1, 4)]
        out = np.empty(12 * sum(sizes), np.float32)
        check(lib().lexp_pairwise_terms(self._h, mode, len(pl), rg.ctypes.data, pl.ctypes.data, out.ctypes.data))
        res, at = [], 0
        for r, n in zip(rg.reshape(-1, 4), sizes):
            blk = out[at:at + 12 * n].reshape(3, 4, int(r[3]), int(r[2]))
            res.append((blk[0], blk[1], blk[2]))
            at += 12 * n
        return res

    def computeDisparities(self, mode=0) -> np.ndarray:
        """StereoEnergy::computeDisparities of the device state (StereoEnergy.h:269-272)."""
        out = np.empty((self.height, self.width), np.float32)
        check(lib().lexp_get_disparities(self._h, mode, out.ctypes.data))
        return out

    def post_process(self, threshold=1.5, fail_out=None):
        """PMStereoBase::postProcess(currentLabeling_[0], currentLabeling_[1], threshold) (PMStereoBase.h:146-256) on the device state of
        both views (pm_begin for each), in place: left-right check, dilation, hole filling, weighted median over windR with the omega of
        set_smoothness.  `fail_out`: optional uint8 [2][H][W] array that receives the fail maps of the check (0 / 128 / 255).
        Returns `fail_out`."""
        if fail_out is not None:
            assert fail_out.dtype == np.uint8 and fail_out.shape == (2, self.height, self.width) and fail_out.flags.c_contiguous
        check(lib().lexp_post_process(self._h, float(threshold), None if fail_out is None else fail_out.ctypes.data))
        return fail_out

    def energy(self, mode=0):
        """(data term, smoothness term) of the device state of view `mode`: sum of currentCost_ and
        StereoEnergy::computeSmoothnessCost(currentLabeling_m) (StereoEnergy.h:165-199)."""
        d, s = C.c_double(0.0), C.c_double(0.0)
        check(lib().lexp_energy(self._h, mode, C.byref(d), C.byref(s)))
        return d.value, s.value

    # --- a whole run: FastGCStereo::run with the Evaluator (lexp_set_ground_truth / lexp_evaluate / lexp_run) ---------------------
    def set_ground_truth(self, gt, nonocc=None):
        """The left view's ground truth for `evaluate` / `run`: float32 [H][W] disparities (0 or inf: none) and the uint8 [H][W]
        non-occlusion mask, of which the pixels equal to 255 count (None: every pixel)."""
        g = np.ascontiguousarray(gt, dtype=np.float32)
        m = None if nonocc is None else np.ascontiguousarray(nonocc, dtype=np.uint8)
        assert g.shape == (self.height, self.width) and (m is None or m.shape == g.shape)
        check(lib().lexp_set_ground_truth(self._h, g.ctypes.data, None if m is None else m.ctypes.data))

    @staticmethod
    def _eval_dict(r) -> dict:
        return {k: getattr(r, k) for k, _ in _capi.EvalResult._fields_}

    def evaluate(self, mode=0, precision=-1.0, threshold=0.5) -> dict:
        """Evaluator::evaluate (Evaluator.h:113-187) on the device state of view `mode` against the left ground truth: energy, data,
        smooth, the pixel counts (valid_pixels, nonocc_pixels, all_correct, nonocc_correct) and the error rates all / nonocc in percent.
        precision > 0 quantises the disparities to multiples of it first."""
        r = _capi.EvalResult()
        check(lib().lexp_evaluate(self._h, int(mode), float(precision), float(threshold), C.byref(r)))
        return self._eval_dict(r)

    def render_evaluation(self, mode=0, precision=-1.0, threshold=0.5):
        """The images Evaluator::evaluate writes for view `mode` (Evaluator.h:123-166, lexp_render_evaluation), rendered on the device:
        (D, N, E) = the quantised disparity * 255 / MAX_DISPARITY as uint8 [H][W], the normal map as uint8 [H][W][3] (BGR) and the error
        map as uint8 [H][W] (255 correct or no ground truth, 200 wrong and occluded, 0 wrong).  set_ground_truth first."""
        H, W = self.height, self.width
        d, n, e = np.empty((H, W), np.uint8), np.empty((H, W, 3), np.uint8), np.empty((H, W), np.uint8)
        check(lib().lexp_render_evaluation(self._h, int(mode), float(precision), float(threshold), d.ctypes.data, n.ctypes.data, e.ctypes.data))
        return d, n, e

    def render_consistency(self):
        """The images of PMStereoBase::viewConsistencyCheck (PMStereoBase.h:87-108, lexp_render_consistency) of both views' device state:
        (C0, C1), uint8 [H][W][3] (BGR) each: the disparity in gray, blue where the other view's pixel is outside the image, red where
        the two views' disparities differ by more than 1.5."""
        H, W = self.height, self.width
        c0, c1 = np.empty((H, W, 3), np.uint8), np.empty((H, W, 3), np.uint8)
        check(lib().lexp_render_consistency(self._h, c0.ctypes.data, c1.ctypes.data))
        return c0, c1

    def run(self, maxIteration, viewModes=(0, 1), pmInit=0, labeling=None, unit_sizes=None, proposers=None, seed=0, precision=-1.0,
            threshold=0.5, callback=None, image_callback=None):
        """FastGCStereo::run(maxIteration, viewModes, pmInit, labeling, rawlabeling) on the device (lexp_run_ex): random start (or the
        given Plane [H][W] labeling), pmInit PatchMatch iterations, maxIteration graph-cut iterations and, with viewModes (0, 1), the
        post-processing.  unit_sizes / proposers: the layers and their [(kind, K)] lists (default: sweep.v3_layer_units and
        sweep.V3_PROPOSERS_REFERENCE).  callback(index, mode, result_dict, seconds) at the Evaluator's points (set_ground_truth first).
        image_callback(index, mode, kind, array) receives the reference's debug images (lexp_run_ex): kind "D", "N", "E" at every
        Evaluator point after `callback`, and with two views "C" of view 0 and view 1 after every iteration and the post-processing;
        the arrays are copies (uint8 [H][W] or [H][W][3] BGR).  Rendering does not count towards `seconds`.
        Returns (labeling, rawlabeling) of view 0, float32 [H][W][4] each."""
        from .sweep import V3_PROPOSERS_REFERENCE, v3_layer_units
        views = tuple(viewModes)
        if views not in ((0,), (0, 1)):
            raise LexpError("viewModes must be (0,) or (0, 1)")
        units = np.ascontiguousarray(unit_sizes if unit_sizes is not None else v3_layer_units(self.width), dtype=np.int32)
        props = proposers if proposers is not None else V3_PROPOSERS_REFERENCE
        n_prop = np.ascontiguousarray([len(p) for p in props], dtype=np.int32)
        kinds = np.ascontiguousarray([k for p in props for k, _ in p], dtype=np.int32)
        Ks = np.ascontiguousarray([K for p in props for _, K in p], dtype=np.int32)
        init = None
        if labeling is not None:
            init = np.ascontiguousarray(labeling, dtype=np.float32)
            assert init.shape == (self.height, self.width, 4)
        o = _capi.RunOptions(len(views), int(pmInit), int(maxIteration), len(units), units.ctypes.data, n_prop.ctypes.data, kinds.ctypes.data,
                             Ks.ctypes.data, None if init is None else init.ctypes.data, int(seed) & 0xFFFFFFFFFFFFFFFF, float(precision),
                             float(threshold))
        lab = np.empty((self.height, self.width, 4), np.float32)
        raw = np.empty((self.height, self.width, 4), np.float32)
        errors = []

        def tramp(_user, index, mode, res, seconds):
            try:
                callback(int(index), int(mode), self._eval_dict(res.contents), float(seconds))
            except BaseException as e:   # an exception cannot cross the C frames: re-raised after the run
                errors.append(e)
        def image_tramp(_user, index, mode, kind, pixels, width, height, channels):
            try:
                shape = (height, width) if channels == 1 else (height, width, channels)
                a = np.ctypeslib.as_array(pixels, shape=shape).copy()
                image_callback(int(index), int(mode), _capi.IMAGE_KINDS[kind], a)
            except BaseException as e:
                errors.append(e)
        cb = _capi.RUN_CALLBACK(tramp) if callback is not None else _capi.RUN_CALLBACK()
        icb = _capi.RUN_IMAGE_CALLBACK(image_tramp) if image_callback is not None else _capi.RUN_IMAGE_CALLBACK()
        check(lib().lexp_run_ex(self._h, C.byref(o), lab.ctypes.data, raw.ctypes.data, cb, icb, None))
        if errors:
            raise errors[0]
        return lab, raw

    # --- PatchMatch phase state: currentCost_[mode] / currentLabeling_[mode] resident on the device ------------------------
    def pm_begin(self, mode=0, cost=None, labeling=None):
        """FastGCStereo::run, :137: currentCost_ = INFINITY (or `cost`), currentLabeling_ = `labeling` (or zeros)."""
        c = None if cost is None else np.ascontiguousarray(cost, dtype=np.float32)
        l = None if labeling is None else np.ascontiguousarray(labeling, dtype=np.float32)
        assert c is None or c.shape == (self.height, self.width)
        assert l is None or l.shape == (self.height, self.width, 4)
        check(lib().lexp_pm_begin(self._h, mode, None if c is None else c.ctypes.data, None if l is None else l.ctypes.data))

    def pm_init_from_labeling(self, mode=0):
        """initCurrentFast started from a given labeling (FastGCStereo.h:116-130): currentCost_[mode](p) = ComputeUnaryPotential(
        (p - windR, 2 windR + 1) & image, {p}, ., currentLabeling_[mode](p)) for every pixel, from the labeling the state holds
        (pm_begin(mode, labeling=...) or written through pm_device_state).  The labeling is unchanged.  Asynchronous on the context's
        stream.  Also recomputes the costs after post_process, which changes only the labels."""
        check(lib().lexp_pm_init_from_labeling(self._h, int(mode)))

    def pm_get(self, mode=0, want_cost=True, want_labeling=True, out_cost=None, out_labeling=None):
        """Copies the state back; `out_cost` / `out_labeling`: caller's (e.g. page-locked) arrays to fill instead of new ones."""
        cost = out_cost if out_cost is not None else (np.empty((self.height, self.width), np.float32) if want_cost else None)
        lab = out_labeling if out_labeling is not None else (np.empty((self.height, self.width, 4), np.float32) if want_labeling else None)
        assert cost is None or (cost.dtype == np.float32 and cost.shape == (self.height, self.width) and cost.flags.c_contiguous)
        assert lab is None or (lab.dtype == np.float32 and lab.shape == (self.height, self.width, 4) and lab.flags.c_contiguous)
        check(lib().lexp_pm_get(self._h, mode, None if cost is None else cost.ctypes.data, None if lab is None else lab.ctypes.data))
        return cost, lab

    # multi-GPU cell shard: every rank's copy of the state is written by all ranks' kernels (peer memory over NVLink)
    def pm_ipc_export(self, mode=0) -> bytes:
        buf = C.create_string_buffer(192)
        check(lib().lexp_pm_ipc_export(self._h, mode, buf))
        return buf.raw

    def pm_ipc_connect(self, rank, world, all_handles, mode=0):
        """all_handles: the `world` exports in rank order (e.g. from torch.distributed.all_gather_object)."""
        blob = b"".join(all_handles)
        assert len(blob) == 192 * world
        check(lib().lexp_pm_ipc_connect(self._h, mode, rank, world, blob))

    def pm_connect_local(self, rank, peers, mode=0):
        """peers: the contexts of all ranks living in this process (tests, single-process multi-device callers)."""
        arr = (C.c_void_p * len(peers))(*[p._h for p in peers])
        check(lib().lexp_pm_connect_local(self._h, mode, rank, len(peers), arr))

    def pm_reset_sync(self):
        check(lib().lexp_pm_reset_sync(self._h))

    def pm_advance_epoch(self, delta, mode=0):
        check(lib().lexp_pm_advance_epoch(self._h, mode, int(delta)))

    def pm_device_state(self, mode=0):
        """(device pointer of currentCost float[H][W], device pointer of currentLabeling Plane[H][W])."""
        a, b = C.c_void_p(), C.c_void_p()
        check(lib().lexp_pm_device_state(self._h, mode, C.byref(a), C.byref(b)))
        return int(a.value), int(b.value)

    def sync(self):
        check(lib().lexp_sync(self._h))

    @property
    def stream(self) -> int:
        return int(lib().lexp_stream(self._h) or 0)

    def set_stream(self, cuda_stream: int):
        """Run on the caller's CUDA stream (e.g. torch.cuda.current_stream().cuda_stream)."""
        check(lib().lexp_set_stream(self._h, C.c_void_p(int(cuda_stream))))

    def set_overlap(self, on=True):
        """Opt in to overlapping launches for eval_device(..., planes_on_device=True): see lexp_set_overlap."""
        check(lib().lexp_set_overlap(self._h, int(bool(on))))

    @property
    def launch_count(self) -> int:
        return int(lib().lexp_launch_count(self._h))

    @property
    def overlapped_launch_count(self) -> int:
        """How many of launch_count carried the programmatic-serialization attribute (may have overlapped their predecessor)."""
        return int(lib().lexp_overlapped_launch_count(self._h))

    @property
    def lean_launch_count(self) -> int:
        """How many of launch_count ran the lean (three CTAs per SM) build of the PatchMatch-phase kernel: see lexp_lean_launch_count."""
        return int(lib().lexp_lean_launch_count(self._h))

    @property
    def combine_stats(self):
        """(batched launches that served concurrent single-cell calls, number of calls they served)."""
        b, n = C.c_int64(0), C.c_int64(0)
        check(lib().lexp_combine_stats(self._h, C.byref(b), C.byref(n)))
        return int(b.value), int(n.value)

    def close(self):
        if getattr(self, "_h", None):
            lib().lexp_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class NaiveStereoEnergy(CostVolumeEnergy):
    """NaiveStereoEnergy (StereoEnergy.h:629-764): the image-based unary term of `-mode MiddV2` (BASELINE.json
    configs[0]) -- 4-channel ExI = [(1-alpha) BGR, alpha d/dx gray], other view warped with cv::warpAffine's fixed-point
    bilinear sampling, truncated L1 colour + gradient cost, aggregated as the reference selects (StereoEnergy.h:666-686): "GF" /
    "GFfloat" (guided filter), "BF" (bilateral filter, sig2 = filter_param1) or "" (none).  No cost volume."""
    ENERGY_KIND = 1
    FILTERS = {"GF": _capi.FILTER_GF, "GFfloat": _capi.FILTER_GF, "BF": _capi.FILTER_BILATERAL, "": _capi.FILTER_NONE}

    def __init__(self, imL, imR, params: Parameters, MAX_DISPARITY, MIN_DISPARITY=0.0, MAX_VDISPARITY=0.0, device: int = 0):
        if imL is None or imR is None:
            raise LexpError("NaiveStereoEnergy needs both images")
        super().__init__(imL, imR, None, None, params, MAX_DISPARITY, MIN_DISPARITY, MAX_VDISPARITY, device)
