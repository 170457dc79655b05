"""Restatements of the two pieces of FastGCStereo::run that the device runs with kernels of their own (lexp_run.cuh): the random start of
initCurrentFast and Evaluator::evaluate.  Test oracle only."""
import numpy as np

from .lexp_oracle import CvRNG, create_random_label, pm_rng_state

f32 = np.float32


def random_start(units, seed, ids, min_disp, max_disp):
    """initCurrentFast with an empty labeling (FastGCStereo.h:100-114) as lexp_pm_sweep_init_random draws it: for unit i,
    selectRandomPixelInRect (FastGCStereo.h:229-236) then StereoEnergy::createRandomLabel (StereoEnergy.h:120-129) from
    CvRNG(pm_rng_state(seed, ids[i])).  Returns float32 [len(units)][4]."""
    out = []
    for (x, y, w, h), cid in zip(units, ids):
        rng = CvRNG(pm_rng_state(seed, int(cid)))
        n = rng.uniform_int(0, w * h)
        out.append(create_random_label(rng, x + n % w, y + n // w, min_disp, max_disp))
    return np.stack(out).astype(np.float32)


def disparities(labeling):
    """computeDisparities (StereoEnergy.h:269-272): a x + b y + c + v 0, every product and sum rounded to float."""
    H, W = labeling.shape[:2]
    L = labeling.astype(np.float32)
    x = np.arange(W, dtype=np.float32)[None, :]
    y = np.arange(H, dtype=np.float32)[:, None]
    with np.errstate(invalid="ignore", over="ignore"):
        return ((L[..., 0] * x + L[..., 1] * y) + L[..., 2]) + L[..., 3] * f32(0.0)


def cv_round(s):
    """cvRound of float64 values as the x86 conversion does it: round half to even, INT_MIN for NaN and for results outside int32."""
    s = np.asarray(s, np.float64)
    ok = (s >= -2147483648.5) & (s < 2147483647.5)
    return np.where(ok, np.rint(np.where(ok, s, 0.0)), -2147483648.0).astype(np.int64).astype(np.int32)


def evaluate_counts(disp, gt, nonocc, precision, threshold):
    """Evaluator::evaluate's error statistics (Evaluator.h:105-110, 124-163) for a float32 disparity map: quantize when precision > 0
    (convertTo CV_32S: d * (float)(1.0 / precision) in float, cvRound; then back with scale precision in double), errorMap = |disp - GT| <= threshold,
    validMask = GT > 0 & GT != inf, the mask pixels = nonocc == 255 (None: all).  Returns (valid, nonocc, all_correct,
    nonocc_correct, all %, nonocc %)."""
    d = np.asarray(disp, np.float32)
    gt = np.asarray(gt, np.float32)
    if precision > 0:
        s = (d * f32(1.0 / np.float64(f32(precision))) + f32(0.0)).astype(np.float32)   # cvtScale 32f -> 32s: float work type
        q = cv_round(s.astype(np.float64))
        d = (q.astype(np.float64) * np.float64(f32(precision))).astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        ok = np.abs(d - gt).astype(np.float64) <= np.float64(f32(threshold))
        valid = (gt > 0) & (gt != np.inf)
    mask = np.ones(gt.shape, bool) if nonocc is None else (np.asarray(nonocc) == 255)
    nv, nn = int(valid.sum()), int(mask.sum())
    ca, cn = int((ok & valid).sum()), int((ok & mask).sum())
    with np.errstate(invalid="ignore", divide="ignore"):
        all_ = (1.0 - np.float64(ca) / np.float64(nv)) * 100.0
        nonocc_ = (1.0 - np.float64(cn) / np.float64(nn)) * 100.0
    return nv, nn, ca, cn, float(all_), float(nonocc_)
