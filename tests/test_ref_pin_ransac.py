"""oracle/ransac_oracle.py against the reference's own RansacProposer (Proposer.h:155-312), compiled from its header into
oracle/_ref/liblexp_ref_ransac.so (oracle/build_ref_ransac.py) over the shim's cv:: layer, whose cv::solve is the contract's double
solve.  The samples' triples are injected into the reference's std::random_shuffle through the library's own rand(), so the
reference runs RANSACPlane's control flow on the oracle's samples: the number of samples drawn, every inlier count (no_i, and no after
each refit) and the plane must be identical."""
import ctypes as C

import numpy as np
import pytest

from oracle import ransac_oracle as RO
import test_gpu_ransac as _gr
from oracle import lexp_oracle as O


def _lib():
    from oracle import build_ref_ransac
    path = build_ref_ransac.build()
    if path is None:
        return None
    L = C.CDLL(path)
    P = C.c_void_p
    L.ref_ransac_run.restype = C.c_int
    L.ref_ransac_run.argtypes = [P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, P, C.c_int, P, P, P, P, C.c_int]
    L.ref_ransac_sample_count.restype = C.c_int
    L.ref_ransac_sample_count.argtypes = [C.c_int, C.c_int]
    L.ref_ransac_shuffle_check.restype = None
    L.ref_ransac_shuffle_check.argtypes = [C.c_int, P, P]
    return L


R = _lib()
if R is None:
    pytest.skip("oracle/_ref/liblexp_ref_ransac.so is not built and the reference's headers are absent", allow_module_level=True)


def ref_run(lab, unit, triples):
    lab = np.ascontiguousarray(lab, np.float32)
    H, W = lab.shape[:2]
    tri = np.ascontiguousarray(triples, np.int32)
    plane = np.zeros(4, np.float32)
    ns = C.c_int(0)
    cap = 2 * RO.MAX_SAM
    counts, owner = np.zeros(cap, np.int32), np.zeros(cap, np.int32)
    n = R.ref_ransac_run(lab.ctypes.data, H, W, *(int(v) for v in unit), tri.ctypes.data, len(tri), plane.ctypes.data, C.byref(ns),
                         counts.ctypes.data, owner.ctypes.data, cap)
    assert n >= 0
    per = [[] for _ in range(ns.value)]
    for c, o in zip(counts[:n], owner[:n]):
        per[o].append(int(c))
    return plane, per


def pin(lab, unit, state):
    """Oracle and reference on the same snapshot and samples: returns the oracle's trace."""
    plane, trace = RO.ransac_proposal(state, lab, unit)
    n = unit[2] * unit[3]
    rng = O.CvRNG(state)
    triples = [RO.draw_triple(rng, n) for _ in range(RO.MAX_SAM)] if n > 3 else [(0, 1, 2)] * RO.MAX_SAM
    ref_plane, ref_per = ref_run(lab, unit, triples)
    assert np.array_equal(ref_plane.view(np.uint32), plane.view(np.uint32)), (unit, ref_plane, plane)
    if n <= 3:   # the oracle draws nothing; the reference's 500 samples cannot exceed 3 inliers
        assert all(c[0] <= 3 and len(c) == 1 for c in ref_per)
        return trace
    assert len(ref_per) == len(trace), (unit, len(ref_per), len(trace))
    for s, (t, r) in enumerate(zip(trace, ref_per)):
        tri, no_i, refit, no, acc, max_sam = t
        assert r == ([no_i, no] if refit else [no_i]), (unit, s, r, t)
    return trace


def test_the_shuffle_interposition_is_in_effect():
    """std::random_shuffle inside the library draws from its rand(): the first three entries are the injected triple."""
    for n, t in ((4, (3, 0, 2)), (5, (1, 0, 2)), (400, (0, 399, 7)), (400, (2, 1, 0)), (34000, (33999, 2, 17)), (7, (6, 5, 4))):
        tri = np.array(t, np.int32)
        out = np.zeros(3, np.int32)
        R.ref_ransac_shuffle_check(n, tri.ctypes.data, out.ctypes.data)
        assert tuple(out) == t, (n, t, tuple(out))


def test_compute_sample_count_equals_the_reference():
    for pt in (4, 5, 10, 37, 400, 3721, 34000, 119025):
        for ni in sorted(set(list(range(0, min(pt, 80) + 1)) + [pt // 3, pt // 2, pt - 1, pt])):
            assert RO.compute_sample_count(ni, pt) == R.ref_ransac_sample_count(ni, pt), (ni, pt)


def test_designed_units():
    """Dyadic plane with outliers, two planes, fronto-parallel, random labels, collinear 1 x k / k x 1 units, n = 3, NaN / inf labels."""
    lab, cases = _gr.designed_scene()
    for seed in (1, 0xDEADBEEF12345678):
        for i, (unit, what) in enumerate(cases):
            if unit[2] * unit[3] < 3:   # the reference reads past its permutation (undefined behaviour)
                continue
            pin(lab, unit, O.pm_rng_state(seed, i))


def test_every_layer0_and_layer1_cell_of_the_cones_crop():
    """The cones crop after one oracle pm iteration (initCurrentFast with random labels, then the device schedule's proposers)."""
    from test_ransac_oracle import cones_state_after_one_pm_iteration
    lab, layers = cones_state_after_one_pm_iteration()
    n_cells = n_samples = n_refits = 0
    for li in (0, 1):
        for r, unit in enumerate(layers[li]["unit"]):
            trace = pin(lab, unit, O.pm_rng_state(77 + li, r))
            n_cells += 1
            n_samples += len(trace)
            n_refits += sum(t[2] for t in trace)
    print(f"{n_cells} cells, {n_samples} samples, {n_refits} refits identical to the reference's")
    assert n_cells > 100 and n_refits > n_cells
