"""Checks of a whole run (lexp_run, DESIGN.md 3h), shared by tests/test_emu_run.py (CPU emulator) and tests/test_gpu_zz_run.py (H100).

The run is certified by composition: lexp_run must equal the same run issued through the public calls it is made of (the sweep object's
random start, pm and graph-cut iterations, lexp_pm_init_from_labeling, lexp_post_process, lexp_evaluate) bit for bit, with the seeds of
sweep.run_seed; each of those calls has its own certification.  The two new kernels are checked against oracle/run_oracle.py."""
import numpy as np

import localexpstereo_b200 as L
from localexpstereo_b200.sweep import RUN_GC, RUN_INIT, RUN_PM, NativePMSweep, run_seed
from oracle import lexp_oracle as O
from oracle import run_oracle as RO
from lexp_testlib import make_scene

SMOOTH = dict(lam=0.6, omega=10.0, th_smooth=1.0, epsilon=0.01)
PROPS = [[(L.PROP_EXPANSION, 1), (L.PROP_RANSAC, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 1), (L.PROP_RANSAC, 1)]]


def scene_energy(H, W, D, windR, naive=False, seed=0):
    imL, imR, volL, volR = make_scene(H, W, D, seed=seed)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.NaiveStereoEnergy(imL, imR, prm, D - 1) if naive else L.CostVolumeEnergy(imL, imR, volL, volR, prm, D - 1)
    E.set_smoothness(**SMOOTH)
    return E


def synthetic_gt(E, seed):
    """A ground truth with every case of the Evaluator: planar disparities, pixels without GT (0 and inf), a mask of 255 / 0 / 128."""
    rng = np.random.default_rng(seed)
    H, W = E.height, E.width
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    gt = (np.float32(0.5) * E.MAX_DISPARITY + np.float32(0.05) * xx - np.float32(0.03) * yy).astype(np.float32)
    gt += rng.normal(0, 1.5, gt.shape).astype(np.float32)
    gt[rng.random(gt.shape) < 0.05] = 0.0
    gt[rng.random(gt.shape) < 0.05] = np.inf
    nonocc = rng.choice(np.array([255, 0, 128], np.uint8), size=gt.shape, p=[0.8, 0.15, 0.05])
    return gt, nonocc


def check_random_start(E, units, seed, exact=True):
    """lexp_pm_sweep_init_random: the labels of the state's unit regions against oracle.run_oracle.random_start.  exact=False: the
    RandomProposer rule of the device (FP64 sin / cos of CUDA against glibc's: 2e-6 relative / 1e-6 absolute, v bit for bit)."""
    S = NativePMSweep(E, unit_sizes=units, proposers=[[(L.PROP_EXPANSION, 1)]] * len(units))
    try:
        S.begin()
        S.random_start(seed)
        cost, lab = S.get()
        lm = L.LayerManager(E.width, E.height, E.params.windR)
        u0 = lm.addLayer(units[0]).unitRegions
        want = RO.random_start(u0, seed, range(len(u0)), E.MIN_DISPARITY, E.MAX_DISPARITY)
        got = np.stack([lab[y, x] for (x, y, w, h) in u0])
        for (x, y, w, h), g in zip(u0, got):   # the unit holds its label everywhere
            assert (lab[y:y + h, x:x + w] == g).all()
        if exact:
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        else:
            assert np.array_equal(got[:, 3], want[:, 3]) and np.allclose(got, want, rtol=2e-6, atol=1e-6), np.abs(got - want).max()
        assert np.isfinite(cost).all()
        return got, want
    finally:
        S.close()


def check_evaluate(E, gt, nonocc, mode=0):
    """lexp_evaluate against numpy on the device's own labeling, for several precisions / thresholds: exact counts and rates."""
    E.set_ground_truth(gt, nonocc)
    _, lab = E.pm_get(mode)
    disp = RO.disparities(lab)
    assert np.array_equal(disp.view(np.uint32), E.computeDisparities(mode).view(np.uint32))
    data, smooth = E.energy(mode)
    for precision, threshold in ((-1.0, 0.5), (0.25, 0.5), (0.5, 1.0), (1.0, 1.0), (0.3, 0.5)):
        r = E.evaluate(mode, precision, threshold)
        want = RO.evaluate_counts(disp, gt, nonocc, precision, threshold)
        got = (r["valid_pixels"], r["nonocc_pixels"], r["all_correct"], r["nonocc_correct"], r["all"], r["nonocc"])
        assert got[:4] == want[:4] and np.array_equal(got[4:], want[4:], equal_nan=True), (precision, threshold, got, want)
        assert (r["data"], r["smooth"], r["energy"]) == (data, smooth, smooth + data)
    a, b = E.evaluate(mode, 0.25, 0.5), E.evaluate(mode, 0.25, 0.5)
    assert np.array_equal(list(a.values()), list(b.values()), equal_nan=True)


def composed_run(E, views, pm, gc, units, props, seed, labeling=None, precision=0.25, threshold=0.5):
    """The run lexp_run makes, issued through the public calls; returns (labeling, raw labeling, [(index, mode, evaluation)])."""
    sw = {m: NativePMSweep(E, unit_sizes=units, proposers=props, mode=m) for m in views}
    pts = []
    ev = lambda i, m: pts.append((i, m, E.evaluate(m, precision, threshold)))
    try:
        for m in views:
            if labeling is None:
                sw[m].begin()
                sw[m].random_start(run_seed(seed, m, RUN_INIT))
            else:
                E.pm_begin(m, None, labeling)
                E.pm_init_from_labeling(m)
            ev(0, m)
        for it in range(pm):
            for m in views:
                sw[m].iteration(it, run_seed(seed, m, RUN_PM, it))
                ev(it + 1, m)
        for it in range(gc):
            for m in views:
                sw[m].gc_iteration(it, run_seed(seed, m, RUN_GC, it))
                ev(it + 1 + pm, m)
        raw = E.pm_get(0)[1]
        if len(views) == 2:
            E.post_process(1.5)
            ev(gc + 1 + pm, 0)
            ev(gc + 1 + pm, 1)
        return E.pm_get(0)[1], raw, pts
    finally:
        for s in sw.values():
            s.close()


def expected_indices(views, pm, gc):
    """The Evaluator's points of FastGCStereo::run (FastGCStereo.h:138,156,182,207-208)."""
    out = [(0, m) for m in views]
    out += [(it + 1, m) for it in range(pm) for m in views]
    out += [(it + 1 + pm, m) for it in range(gc) for m in views]
    if len(views) == 2:
        out += [(gc + 1 + pm, 0), (gc + 1 + pm, 1)]
    return out


def check_run_equals_composition(mk, views, pm, gc, units, props, seed, given=False):
    """lexp_run against composed_run on two contexts built by mk(): labelings bit for bit, the callback at exactly the reference's
    indices with the composition's evaluations, non-decreasing positive times."""
    Ea, Eb = mk(), mk()
    try:
        gt, nonocc = synthetic_gt(Ea, seed)
        Ea.set_ground_truth(gt, nonocc)
        Eb.set_ground_truth(gt, nonocc)
        labeling = None
        if given:
            rng = O.CvRNG(seed)
            lm = L.LayerManager(Ea.width, Ea.height, Ea.params.windR)
            labeling = np.zeros((Ea.height, Ea.width, 4), np.float32)
            for (x, y, w, h) in lm.addLayer(units[-1]).unitRegions:
                labeling[y:y + h, x:x + w] = O.create_random_label(rng, x, y, Ea.MIN_DISPARITY, Ea.MAX_DISPARITY)
        calls = []
        lab, raw = Ea.run(gc, views, pm, labeling, units, props, seed, 0.25, 0.5, callback=lambda i, m, r, t: calls.append((i, m, r, t)))
        lab_c, raw_c, pts = composed_run(Eb, views, pm, gc, units, props, seed, labeling)
        assert [(i, m) for i, m, _, _ in calls] == expected_indices(views, pm, gc)
        assert [(i, m) for i, m, _ in pts] == expected_indices(views, pm, gc)
        for (_, _, r, _), (_, _, rc) in zip(calls, pts):
            assert r == rc, (r, rc)
        times = [t for *_, t in calls]
        assert times[0] == 0.0 and all(b >= a for a, b in zip(times, times[1:])) and times[-1] > 0.0
        assert np.array_equal(lab.view(np.uint32), lab_c.view(np.uint32))
        assert np.array_equal(raw.view(np.uint32), raw_c.view(np.uint32))
        if len(views) == 1:
            assert np.array_equal(lab, raw)
        return lab, raw, calls
    finally:
        Ea.close(); Eb.close()
