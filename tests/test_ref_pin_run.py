"""The oracles of a whole run (oracle/run_oracle.py) against the reference's own code, compiled from its headers into
oracle/_ref/liblexp_ref_run.so (oracle/build_ref_run.py): the random start (selectRandomPixelInRect + StereoEnergy::createRandomLabel
from the same cv::theRNG() state) bit for bit, and the Evaluator (Evaluator::evaluate of the real Evaluator.h) on designed labelings --
quantisation ties at (k + 0.5) * precision for power-of-two and other precisions, GT 0 and inf, empty and full masks, precision -1."""
import numpy as np
import pytest

from oracle import lexp_oracle as O
from oracle import ref_run
from oracle import run_oracle as RO

if not ref_run.available():
    pytest.skip("oracle/_ref/liblexp_ref_run.so is not built and the reference's headers are absent", allow_module_level=True)

H, W = 36, 52
IM_L = O.synthetic_image(H, W, 5)
IM_R = O.synthetic_image(H, W, 6)


@pytest.mark.parametrize("seed", [0, 1, 2**40 + 7, 2**64 - 1])
def test_random_start_equals_the_reference(seed):
    rng = np.random.default_rng(seed % 1000)
    units = [(int(rng.integers(0, W - 12)), int(rng.integers(0, H - 12)), int(rng.integers(1, 12)), int(rng.integers(1, 12))) for _ in range(200)]
    ids = np.arange(len(units)) * 7 + 3
    states = [O.pm_rng_state(seed, int(i)) for i in ids]
    for max_disp in (15.0, 58.0):
        want = ref_run.random_start(IM_L, IM_R, max_disp, units, states)
        got = RO.random_start(units, seed, ids, 0.0, max_disp)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def tie_labeling(precision, rng):
    """Constant planes (a = b = v = 0) whose disparity c sits on quantisation ties (k + 0.5) * precision in float, next to them, and at random."""
    p = np.float32(precision) if precision > 0 else np.float32(0.25)
    k = rng.integers(0, 200, (H, W)).astype(np.float32)
    c = ((k + np.float32(0.5)) * p).astype(np.float32)
    pick = rng.random((H, W))
    c = np.where(pick < 0.15, np.nextafter(c, np.float32(np.inf)), c)
    c = np.where((pick >= 0.15) & (pick < 0.3), np.nextafter(c, np.float32(-np.inf)), c)
    c = np.where(pick >= 0.8, rng.uniform(0, 60, (H, W)).astype(np.float32), c).astype(np.float32)
    lab = np.zeros((H, W, 4), np.float32)
    lab[..., 2] = c
    return lab


def gt_for(lab, rng):
    gt = (lab[..., 2] + rng.choice(np.float32([0.0, 0.25, 0.5, -0.5, 0.75, 1.0]), (H, W))).astype(np.float32)
    gt[rng.random((H, W)) < 0.1] = 0.0
    gt[rng.random((H, W)) < 0.1] = np.inf
    return gt


@pytest.mark.parametrize("precision", [0.25, 0.3, float(np.float32(1 / 3)), 0.125, 1.0, -1.0])
@pytest.mark.parametrize("mask", ["mixed", "empty", "full"])
def test_evaluator_equals_the_reference(precision, mask):
    rng = np.random.default_rng(int(abs(precision) * 1000) + len(mask))
    lab = tie_labeling(precision, rng)
    gt = gt_for(lab, rng)
    nonocc = {"mixed": np.where(rng.random((H, W)) < 0.7, 255, 0), "empty": np.zeros((H, W)), "full": np.full((H, W), 255)}[mask].astype(np.uint8)
    cost = rng.uniform(0, 3, (H, W)).astype(np.float32)
    for threshold in (0.5, 1.0):
        ref = ref_run.evaluate(IM_L, IM_R, 58.0, lab, cost, gt, nonocc, precision, threshold)
        nv, nn, ca, cn, all_, nonocc_ = RO.evaluate_counts(RO.disparities(lab), gt, nonocc, precision, threshold)
        assert (nv, nn) == (ref["valid_pixels"], ref["nonocc_pixels"])
        assert all_ == ref["all"]
        assert "%f" % all_ == "%f" % ref["log_all"] and "%f" % nonocc_ == "%f" % ref["log_nonocc"], (all_, nonocc_, ref)


def test_double_and_float_quantisation_differ_where_the_reference_follows_float():
    """precision 0.3f, d = 23.25: d * (float)(1 / 0.3f) rounds to 78 in float and to 77 in double; the reference counts it as 78 * 0.3."""
    lab = np.zeros((H, W, 4), np.float32)
    lab[..., 2] = np.float32(23.25)
    gt = np.full((H, W), np.float32(78 * np.float64(np.float32(0.3))), np.float32)
    ref = ref_run.evaluate(IM_L, IM_R, 58.0, lab, np.zeros((H, W), np.float32), gt, np.full((H, W), 255, np.uint8), 0.3, 0.0)
    assert ref["all"] == 0.0
    assert RO.evaluate_counts(RO.disparities(lab), gt, None, 0.3, 0.0)[4] == 0.0
