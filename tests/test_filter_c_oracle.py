"""The C oracle's batched bilateral / unfiltered path of the cost-volume energy (COracle.filter_unary_batch, oracle/lexp_oracle.c)
against the numpy oracle oracle/filter_oracle.py, which tests/test_ref_pin_filters.py pins to the compiled reference: filterRects at
every corner, inside the image and over all of it, 1x1 and larger targets, steep / NaN / +-inf planes, both views, with and without the
check, windR 2 / 5 / 20 / 21, MIN_DISPARITY != 0.  "" bit for bit; bilateral q within 1e-12 max(sum w |p|, 1e-3) and sum w |p| within
1e-12 relative (both FP64, only the order of the sums may differ); the NaN and COST_FOR_INVALID patterns exactly.  The C path is the
(Q) oracle of every target pixel of the filter sweeps (tests/pm_step_rig.py)."""
import numpy as np
import pytest

from oracle import c_oracle
from oracle import lexp_oracle as O
import filter_checks as FC
from lexp_testlib import bits, make_scene

REL = 1e-12


def c_oracle_for(scene, windR, MIN, MAX):
    imL, imR, volL, volR = scene
    H, W = imL.shape[:2]
    C = c_oracle.COracle(H, W, volL.shape[0], windR, 1e-4, 0.5, MAX, MIN)
    for m, (im, vol) in enumerate(((imL, volL), (imR, volR))):
        C.set_image(m, im)
        C.set_volume(m, vol)
    return C


def check(H, W, D, windR, filt, mode, seed, MIN=0.0, MAX=None, sig2=10.0):
    scene = make_scene(H, W, D, seed)
    MAX = float(D - 1 if MAX is None else MAX)
    Or = FC.make_oracle("cv", filt, scene, windR, MIN, MAX, sig2)
    C = c_oracle_for(scene, windR, MIN, MAX)
    kind = C.FILTER_BILATERAL if filt == "bl" else C.FILTER_NONE
    try:
        fr, tr = FC.corner_calls(H, W, windR)
        planes = FC.plan_planes(len(fr), H, W, MIN, MAX, 900 + seed)
        planes[2] = np.float32([0.0, 0.0, -np.inf, 0.0])       # -inf
        for wc in (True, False):
            # one call per batch: corner_calls' targetRects overlap the whole-image call's
            for i, (f, t) in enumerate(zip(fr, tr)):
                q, s = C.filter_unary_batch(mode, [f], [t], [planes[i]], with_check=wc, filter=kind, windR=windR, sig2=sig2)
                x, y, w, h = t
                q, s = q[y:y + h, x:x + w], s[y:y + h, x:x + w]
                rq, rs = Or.unary(tuple(f), tuple(t), planes[i], mode, with_check=wc)
                what = f"{filt} windR {windR} mode {mode} call {i} check {wc}"
                nan = np.isnan(rq)
                assert np.array_equal(np.isnan(q), nan), f"{what}: NaN pattern of q"
                assert np.array_equal(q == O.COST_FOR_INVALID, rq == O.COST_FOR_INVALID), f"{what}: COST_FOR_INVALID mask"
                assert np.array_equal(np.isnan(s), np.isnan(rs)), f"{what}: NaN pattern of sum w |p|"
                if filt == "none":
                    assert np.array_equal(bits(q), bits(rq)) and np.array_equal(bits(s), bits(rs)), what
                    continue
                k = ~nan
                assert (np.abs(q[k] - rq[k]) <= REL * np.maximum(rs[k], 1e-3)).all(), what
                k = ~np.isnan(rs) & np.isfinite(rs)
                assert (np.abs(s[k] - rs[k]) <= REL * np.abs(rs[k])).all(), what
                assert np.array_equal(s[~k & ~np.isnan(rs)], rs[~k & ~np.isnan(rs)]), what
        # the whole batch at once writes exactly the targetRects of its (disjoint) calls
        keep = [0, 1, 2, 3]
        q, s = C.filter_unary_batch(mode, fr[keep], tr[keep], planes[keep], filter=kind, windR=windR, sig2=sig2)
        inside = np.zeros((H, W), bool)
        for i in keep:
            x, y, w, h = tr[i]
            inside[y:y + h, x:x + w] = True
            q1 = C.filter_unary_batch(mode, [fr[i]], [tr[i]], [planes[i]], filter=kind, windR=windR, sig2=sig2)[0]
            assert np.array_equal(bits(q[y:y + h, x:x + w]), bits(q1[y:y + h, x:x + w])), "a batch differs from its single calls"
        assert np.isnan(q[~inside]).all() and np.isnan(s[~inside]).all(), "a pixel outside the targetRects was written"
    finally:
        C.close()


@pytest.mark.parametrize("filt", ["bl", "none"])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("windR", [2, 5, 20, 21])
def test_c_oracle_equals_numpy_oracle(filt, mode, windR):
    check(47, 61, 10, windR, filt, mode, seed=windR + mode)


@pytest.mark.parametrize("filt", ["bl", "none"])
@pytest.mark.parametrize("mode", [0, 1])
def test_c_oracle_min_disparity(filt, mode):
    check(30, 44, 14, 5, filt, mode, seed=3, MIN=2.0, MAX=9.5)
    check(30, 44, 14, 5, filt, mode, seed=4, MIN=-3.0, MAX=8.0)


def test_c_oracle_sig2():
    """sig2 is the reference's float filter_param1: a value that float rounds; a small one that makes most weights tiny."""
    check(31, 40, 8, 5, "bl", 0, seed=7, sig2=0.7)
    check(31, 40, 8, 5, "bl", 1, seed=8, sig2=2.5)


def test_c_oracle_refuses():
    C = c_oracle_for(make_scene(8, 10, 4), 2, 0.0, 3.0)
    try:
        f = np.int32([[0, 0, 10, 8]])
        for kind, sig2 in ((0, 10.0), (3, 10.0), (C.FILTER_BILATERAL, 0.0), (C.FILTER_BILATERAL, -1.0), (C.FILTER_BILATERAL, np.nan)):
            with pytest.raises(ValueError):
                C.filter_unary_batch(0, f, f, np.zeros((1, 4), np.float32), filter=kind, windR=2, sig2=sig2)
    finally:
        C.close()
