"""Restatement of the reference's debug images (DESIGN.md 3j): the Evaluator's D / N / E images (Evaluator.h:123-166) and the images of
viewConsistencyCheck (PMStereoBase.h:87-108), with OpenCV's float evaluation order and imwrite's conversion of a float image to 8 bits.
Test oracle only.  Every array operation is on float32, so each product and sum is rounded to float as OpenCV rounds it."""
import numpy as np

from .run_oracle import cv_round, disparities

f32 = np.float32


def sat8(v):
    """saturate_cast<uchar>(float) on x86-64, the conversion imwrite and convertTo(CV_8U) apply: cvRound of the float (round half to even;
    NaN and values outside int32 give INT_MIN), then clamp to 0 .. 255."""
    v = np.asarray(v, np.float32)
    with np.errstate(invalid="ignore"):
        ok = (v >= f32(-2147483648.0)) & (v < f32(2147483648.0))
    r = np.where(ok, np.rint(np.where(ok, v, f32(0.0)).astype(np.float64)), 0.0)
    return np.clip(r, 0, 255).astype(np.uint8)


def quantized_disparities(labeling, precision):
    """Evaluator::evaluate's disp: computeDisparities, then quantize when precision > 0 (as run_oracle.evaluate_counts)."""
    d = disparities(labeling).astype(np.float32)
    if precision > 0:
        with np.errstate(invalid="ignore", over="ignore"):
            s = (d * f32(1.0 / np.float64(f32(precision))) + f32(0.0)).astype(np.float32)
        d = (cv_round(s.astype(np.float64)).astype(np.float64) * np.float64(f32(precision))).astype(np.float32)
    return d


def d_float(labeling, precision, max_disp):
    """disparityMapVis * 255 as the float image imwrite receives: disp * DISPARITY_FACTOR / 255 is one convertTo with scale
    (double)F * (1.0 / 255) applied in float, F = 255.0f / max_disp (main.cpp:291,380); * 255 is a second float convertTo."""
    alpha = f32(np.float64(f32(255.0) / f32(max_disp)) * (1.0 / 255))
    d = quantized_disparities(labeling, precision)
    with np.errstate(invalid="ignore", over="ignore"):
        return ((d * alpha + f32(0.0)) * f32(255.0)).astype(np.float32)


def n_float(labeling):
    """normalMapVis * 255 (StereoEnergy::computeNormalMap, StereoEnergy.h:274-289): BGR = (nz, (-b nz + 1) / 2, (-a nz + 1) / 2) * 255,
    nz = 1 / sqrt(a a + b b + 1), every operation rounded to float.  float32 [H][W][3]."""
    a = labeling[..., 0].astype(np.float32)
    b = labeling[..., 1].astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        nz = f32(1.0) / np.sqrt((a * a + b * b) + f32(1.0))
        g = (-(b * nz) + f32(1.0)) / f32(2.0)
        r = (-(a * nz) + f32(1.0)) / f32(2.0)
        return np.stack([nz * f32(255.0), g * f32(255.0), r * f32(255.0)], axis=-1).astype(np.float32)


def e_image(labeling, gt, nonocc, precision, threshold):
    """errorMapVis (Evaluator.h:131-133): 255 where |disp - GT| <= threshold or GT is invalid (0 or inf), else 200 where occluded
    (valid GT, nonocc != 255), else 0.  nonocc: the uint8 mask as set_ground_truth takes it (None: every pixel non-occluded)."""
    d = quantized_disparities(labeling, precision)
    gt = np.asarray(gt, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        ok = np.abs(d - gt).astype(np.float64) <= np.float64(f32(threshold))
        valid = (gt > 0) & (gt != np.inf)
    nocc = np.ones(gt.shape, bool) if nonocc is None else (np.asarray(nonocc) == 255)
    return np.where(ok | ~valid, 255, np.where(nocc, 0, 200)).astype(np.uint8)


def eval_images(labeling, gt, nonocc, precision, threshold, max_disp):
    """(D, N, E) of one view as Evaluator::evaluate writes them: uint8 [H][W], [H][W][3] (BGR), [H][W]."""
    return sat8(d_float(labeling, precision, max_disp)), sat8(n_float(labeling)), e_image(labeling, gt, nonocc, precision, threshold)


def consistency_fail(disp0, disp1, threshold=1.5):
    """doConsistencyCheck (PMStereoBase.h:111-144) of two float32 disparity maps: fail [2][H][W] = 0 consistent, 255 the other view's
    disparity at rx = int(x -+ d + 0.5f) differs by more than threshold, 128 rx outside the image (or not an int32)."""
    H, W = disp0.shape
    x = np.arange(W, dtype=np.float32)[None, :]
    out = np.empty((2, H, W), np.uint8)
    for i, (me, other) in enumerate(((disp0, disp1), (disp1, disp0))):
        with np.errstate(invalid="ignore", over="ignore"):
            v = (x - me * f32(-1.0 if i else 1.0)) + f32(0.5)
            inside = (v > f32(-2147483648.0)) & (v < f32(2147483648.0))
            rx = np.where(inside, np.trunc(np.where(inside, v, f32(0.0))), -1.0).astype(np.int64)
            inside &= (rx >= 0) & (rx < W)
            rxc = np.clip(rx, 0, W - 1)
            dsr = np.take_along_axis(other, rxc, axis=1)
            bad = np.abs(dsr - me) > f32(threshold)
        out[i] = np.where(inside, np.where(bad, 255, 0), 128)
    return out


def check_images(lab0, lab1, min_disp, max_disp):
    """(C0, C1) of viewConsistencyCheck: gray = saturate_cast<uchar>(disp * s + o) with s = 255.0f / (max_disp - min_disp),
    o = -min_disp * s (float convertTo), BGR = (fail == 128 ? 255 : gray, gray, fail == 255 ? 255 : gray).  uint8 [H][W][3] each."""
    s = f32(255.0) / (f32(max_disp) - f32(min_disp))
    o = -f32(min_disp) * s
    disp = [disparities(lab0).astype(np.float32), disparities(lab1).astype(np.float32)]
    fail = consistency_fail(disp[0], disp[1])
    out = []
    for m in range(2):
        with np.errstate(invalid="ignore", over="ignore"):
            gray = sat8(disp[m] * s + o)
        out.append(np.stack([np.where(fail[m] == 128, 255, gray), gray, np.where(fail[m] == 255, 255, gray)], axis=-1).astype(np.uint8))
    return out[0], out[1]
