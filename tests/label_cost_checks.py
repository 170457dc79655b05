"""Checks of lexp_pm_init_from_labeling (initCurrentFast started from a given labeling, FastGCStereo.h:116-130), shared by
tests/test_gpu_label_cost.py and tests/test_emu_label_cost.py: designed plane fields, the per-pixel filterRects F(p), and the
oracles the device costs are held against.

For every pixel p the expected cost is ComputeUnaryPotential(F(p), {p}, ., L(p)) with F(p) = (p - windR, 2 windR + 1) & image:
  * cost-volume energy: the FP64 C oracle (oracle_unary_batch), one 1x1 call per pixel with F(p) as its filterRect;
  * both energies: the compiled reference itself (ref_pm_init with one 1x1 unit per pixel, exactly the reference's branch) where
    oracle/_ref is built, and the numpy restatement of NaiveStereoEnergy for the image-based energy.
The labeling must come back unchanged bit for bit; the COST_FOR_INVALID and NaN patterns must match exactly and every other cost
within |d| <= 1e-4 max(|ref|, 1e-3)."""
import numpy as np

from oracle import build_ref
from oracle import c_oracle
from oracle import lexp_oracle as O
from lexp_testlib import assert_costs_close, bits


def all_pixels(H, W):
    ys, xs = np.mgrid[0:H, 0:W]
    return ys.ravel(), xs.ravel()


def filter_rects(H, W, windR, ys, xs):
    """F(p) = (x - windR, y - windR, 2 windR + 1, 2 windR + 1) & image, int32 [n][4]"""
    x0, y0 = np.maximum(xs - windR, 0), np.maximum(ys - windR, 0)
    x1, y1 = np.minimum(xs + windR + 1, W), np.minimum(ys + windR + 1, H)
    return np.stack([x0, y0, x1 - x0, y1 - y0], 1).astype(np.int32)


def random_plane_field(H, W, lo, hi, seed, v=False, slope=0.4, beyond=0.3, nonfinite=0.0):
    """Independent random planes per pixel (the worst case for locality): disparity at the pixel uniform in
    [lo - beyond span, hi + beyond span], so both clamps of the sampler and invalid labels occur, slopes in [-slope, slope].
    v: a non-zero 4th component; nonfinite: the fraction of planes with a NaN or +-inf component."""
    rng = np.random.default_rng(seed)
    span = hi - lo
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float32)
    z = rng.uniform(lo - beyond * span, hi + beyond * span, (H, W)).astype(np.float32)
    a = rng.uniform(-slope, slope, (H, W)).astype(np.float32)
    b = rng.uniform(-slope, slope, (H, W)).astype(np.float32)
    c = (z - a * xs - b * ys).astype(np.float32)
    vv = rng.uniform(-2.0, 2.0, (H, W)).astype(np.float32) if v else np.zeros((H, W), np.float32)
    lab = np.ascontiguousarray(np.stack([a, b, c, vv], -1), np.float32)
    if nonfinite:
        n = max(1, int(nonfinite * H * W))
        idx = rng.choice(H * W, size=min(n, H * W), replace=False)
        vals = np.array([np.nan, np.inf, -np.inf], np.float32)
        flat = lab.reshape(-1, 4)
        flat[idx, rng.integers(0, 3, len(idx))] = vals[rng.integers(0, 3, len(idx))]
    return lab


def painted_field(units, labels, H, W):
    """One label painted over each unit region (the state initCurrentFast's random branch leaves)."""
    lab = np.zeros((H, W, 4), np.float32)
    for (x, y, w, h), p in zip(units, labels):
        lab[y:y + h, x:x + w] = p
    return lab


def device_costs(E, labeling, mode=0):
    """pm_begin with the labeling, then the call under test; checks the labeling is unchanged."""
    E.pm_begin(mode, labeling=labeling)
    E.pm_init_from_labeling(mode)
    cost, lab = E.pm_get(mode)
    assert np.array_equal(bits(lab), bits(labeling)), "the labeling changed"
    return cost


def compare(got, ref, what=""):
    """NaN and COST_FOR_INVALID patterns exact, the rest within the tolerance; returns the worst relative error."""
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), f"{what}: NaN pattern differs at {np.argwhere(np.isnan(got) != np.isnan(ref))[:5]}"
    keep = ~np.isnan(ref)
    return assert_costs_close(got[keep], ref[keep], what)


def c_oracle_costs(im, vol, windR, labeling, ys, xs, mode=0, MIN=0.0, MAX=None, th_col=0.5, nthreads=16):
    """The FP64 C oracle of the cost-volume energy: one ComputeUnaryPotential(F(p), {p}) per pixel (ys, xs).  Returns [n].
    Each pixel is its own oracle_unary call (fresh scratch: the F(p) of neighbouring pixels have different shapes), spread over
    host threads (ctypes releases the GIL)."""
    import ctypes as C
    from concurrent.futures import ThreadPoolExecutor
    D, H, W = vol.shape
    MAX = float(D - 1 if MAX is None else MAX)
    Cc = c_oracle.COracle(H, W, D, windR, 1e-4, th_col, MAX, MIN)
    try:
        Cc.set_image(mode, im)
        Cc.set_volume(mode, vol)
        fr = filter_rects(H, W, windR, ys, xs)
        tr = np.ascontiguousarray(np.stack([xs, ys, np.ones_like(xs), np.ones_like(xs)], 1), np.int32)
        pl = np.ascontiguousarray(labeling[ys, xs], np.float32)
        out = np.full(len(ys), np.nan, np.float32)
        f = c_oracle.lib().oracle_unary
        stride = 4 * 4

        def run(lo_hi):
            for i in range(*lo_hi):
                f(Cc._h, mode, fr.ctypes.data + i * stride, tr.ctypes.data + i * stride, pl.ctypes.data + i * stride,
                  out.ctypes.data + 4 * i, 1, 1)
        n = len(ys)
        chunks = [(k * n // nthreads, (k + 1) * n // nthreads) for k in range(nthreads)]
        with ThreadPoolExecutor(nthreads) as ex:
            list(ex.map(run, chunks))
        return out
    finally:
        Cc.close()


def naive_oracle_costs(Or, windR, labeling, ys, xs, mode=0):
    """The numpy NaiveStereoEnergy oracle, one call per pixel (small scenes only).  Returns [n]."""
    H, W = labeling.shape[:2]
    fr = filter_rects(H, W, windR, ys, xs)
    return np.array([Or.compute_unary_potential(tuple(f), (int(x), int(y), 1, 1), labeling[y, x], mode)[0, 0]
                     for f, y, x in zip(fr, ys, xs)], np.float32)


def reference_available():
    return build_ref.available()


def reference_costs(scene, windR, labeling, mode=0, naive=False, MIN=0.0, MAX=None, nthreads=16, **prm):
    """The compiled reference's own initCurrentFast branch: ref_pm_init with one 1x1 unit per pixel.  Returns [H][W]."""
    from oracle import ref_binding as R
    imL, imR, volL, volR = scene
    H, W = imL.shape[:2]
    if naive:
        D = int(MAX) + 1
        ref = R.RefEnergy(imL, imR, windR=windR, eps=1e-4, th_col=prm.get("th_col", 10.0), th_grad=prm.get("th_grad", 2.0),
                          alpha=prm.get("alpha", 0.9), max_disp=float(MAX), min_disp=MIN, kind=1)
    else:
        D = volL.shape[0]
        ref = R.RefEnergy(imL, imR, volL, volR, windR=windR, eps=1e-4, th_col=prm.get("th_col", 0.5),
                          max_disp=float(D - 1 if MAX is None else MAX), min_disp=MIN, kind=0)
    try:
        ys, xs = all_pixels(H, W)
        units = np.stack([xs, ys, np.ones_like(xs), np.ones_like(xs)], 1).astype(np.int32)
        cost = np.full((H, W), np.nan, np.float32)
        lab = np.zeros((H, W, 4), np.float32)
        ref.pm_init(units, labeling.reshape(-1, 4), windR, cost, lab, mode=mode, nthreads=nthreads)
        assert np.array_equal(bits(lab), bits(labeling))
        return cost
    finally:
        ref.close()


def check_cost_volume_scene(H, W, D, windR, mode=0, MIN=0.0, MAX=None, seed=0, nonfinite=0.02, with_reference=True):
    """Independent random planes (beyond both ends of [MIN, MAX], some NaN / inf) on a synthetic scene: every pixel against the C
    oracle, and against the compiled reference where it is built.  Returns the worst relative error."""
    import localexpstereo_b200 as L
    from lexp_testlib import make_scene
    scene = make_scene(H, W, D, seed)
    imL, imR, volL, volR = scene
    MAX = float(D - 1 if MAX is None else MAX)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.CostVolumeEnergy(imL, imR, volL, volR, prm, MAX, MIN)
    try:
        lab = random_plane_field(H, W, MIN, MAX, 100 + seed, nonfinite=nonfinite)
        got = device_costs(E, lab, mode)
        again = device_costs(E, lab, mode)
        assert np.array_equal(bits(got), bits(again)), "two calls differ"
        ys, xs = all_pixels(H, W)
        ref = c_oracle_costs(imR if mode else imL, volR if mode else volL, windR, lab, ys, xs, mode, MIN, MAX)
        worst = compare(got[ys, xs], ref, f"C oracle {H}x{W} windR {windR} mode {mode}")
        assert (ref == O.COST_FOR_INVALID).any() and (ref != O.COST_FOR_INVALID).any()
        if with_reference and reference_available():
            worst = max(worst, compare(got, reference_costs(scene, windR, lab, mode, MIN=MIN, MAX=MAX), "reference"))
        return worst
    finally:
        E.close()


def check_naive_scene(H, W, D, windR, mode=0, seed=0, with_reference=True):
    """The image-based energy with independent random planes with v != 0: every pixel against the numpy oracle, and against the
    compiled reference where it is built."""
    from lexp_testlib import energy_and_oracle, make_scene
    scene = make_scene(H, W, D, seed)
    E, Or = energy_and_oracle(scene, D, windR, mode, naive=True)
    try:
        lab = random_plane_field(H, W, 0.0, D - 1.0, 200 + seed, v=True, nonfinite=0.02)
        got = device_costs(E, lab, mode)
        ys, xs = all_pixels(H, W)
        worst = compare(got[ys, xs], naive_oracle_costs(Or, windR, lab, ys, xs, mode), f"naive oracle {H}x{W} windR {windR} mode {mode}")
        if with_reference and reference_available():
            worst = max(worst, compare(got, reference_costs(scene, windR, lab, mode, naive=True, MAX=D - 1.0), "naive reference"))
        return worst
    finally:
        E.close()


def check_argument_errors():
    """LEXP_ERR_STATE before pm_begin, LEXP_ERR_INVALID for a bad mode; neither enqueues anything."""
    import localexpstereo_b200 as L
    from lexp_testlib import make_scene
    import pytest
    imL, imR, volL, volR = make_scene(12, 16, 6)
    prm = L.Parameters(windR=4, filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.CostVolumeEnergy(imL, imR, volL, volR, prm, 5)
    try:
        n0 = E.launch_count
        with pytest.raises(L.LexpError, match="lexp error -3: lexp_pm_begin"):
            E.pm_init_from_labeling(0)
        E.pm_begin(0)
        E.sync()
        n0 = E.launch_count
        for bad in (-1, 2):
            with pytest.raises(L.LexpError, match="lexp error -1"):
                E.pm_init_from_labeling(bad)
        with pytest.raises(L.LexpError, match="lexp error -3: lexp_pm_begin"):
            E.pm_init_from_labeling(1)   # view 1 has no state yet
        assert E.launch_count == n0
    finally:
        E.close()
