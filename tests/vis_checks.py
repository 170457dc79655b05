"""Checks of the reference's debug images on the device (lexp_vis.cuh, DESIGN.md 3j), shared by tests/test_emu_vis.py (CPU emulator)
and tests/test_gpu_vis.py (H100).

lexp_render_evaluation / lexp_render_consistency are held bit for bit against oracle/vis_oracle.py on designed states; lexp_run_ex is
held against the run composed of the public calls (as run_checks.composed_run issues it), rendered at every point of the reference."""
import numpy as np

import localexpstereo_b200 as L
from localexpstereo_b200._capi import check, lib
from localexpstereo_b200.sweep import RUN_GC, RUN_INIT, RUN_PM, NativePMSweep, run_seed
from oracle import vis_oracle as V
import run_checks as RC

f32 = np.float32
PRECISIONS = ((-1.0, 0.5), (0.25, 0.5), (0.3, 1.0))   # none, a power of two (and the cones pair's gt_prec), any other


def designed_labeling(H, W, max_disp, seed):
    """A Plane [H][W] labeling with every case of the images, pixel by pixel: ordinary planes, fronto-parallel disparities on k + 0.5 and
    one ulp either side, negative disparities and disparities above max_disp, a = b = 0 (N's G and R = 127.5), steep planes, NaN / inf
    coefficients and v, huge disparities (outside int32 after scaling)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    lab = np.zeros((H, W, 4), np.float32)
    kind = rng.integers(0, 8, size=(H, W))
    a = rng.uniform(-0.4, 0.4, (H, W)).astype(np.float32)
    b = rng.uniform(-0.4, 0.4, (H, W)).astype(np.float32)
    d = rng.uniform(-4.0, max_disp + 4.0, (H, W)).astype(np.float32)
    lab[..., 0], lab[..., 1] = a, b
    lab[..., 2] = d - a * xx - b * yy                                            # 0: an ordinary plane through d at (x, y)
    half = (rng.integers(-3, int(max_disp) + 4, (H, W)) + f32(0.5)).astype(np.float32)
    for k, c in ((1, half), (2, np.nextafter(half, f32(np.inf))), (3, np.nextafter(half, f32(-np.inf)))):
        sel = kind == k
        lab[sel, 0] = 0.0
        lab[sel, 1] = 0.0
        lab[sel, 2] = c[sel]
    sel = kind == 4                                                               # steep planes
    lab[sel, 0] = rng.choice([-1, 1], sel.sum()) * rng.uniform(1.0, 60.0, sel.sum())
    lab[sel, 1] = rng.choice([-1, 1], sel.sum()) * rng.uniform(1.0, 60.0, sel.sum())
    sel = np.argwhere(kind == 5)                                                  # NaN / inf
    specials = [(0, np.nan), (1, np.nan), (2, np.nan), (3, np.nan), (0, np.inf), (1, -np.inf), (2, np.inf), (2, -np.inf), (2, 3e9), (2, -3e9)]
    for i, (y, x) in enumerate(sel):
        ch, v = specials[i % len(specials)]
        lab[y, x, ch] = v
    return lab


def designed_gt(H, W, max_disp, lab, seed):
    """GT near the labeling's disparities on a third of the pixels (correct ones), far elsewhere; 0 and inf; a 255 / 0 / 128 mask."""
    rng = np.random.default_rng(seed + 1)
    with np.errstate(invalid="ignore", over="ignore"):
        disp = V.disparities(lab)
    gt = rng.uniform(0.5, max_disp, (H, W)).astype(np.float32)
    near = (rng.random((H, W)) < 0.35) & np.isfinite(disp) & (np.abs(disp) < 1e6)
    gt[near] = np.maximum(disp[near] + rng.uniform(-0.7, 0.7, near.sum()).astype(np.float32), f32(0.01))
    gt[rng.random((H, W)) < 0.08] = 0.0
    gt[rng.random((H, W)) < 0.08] = np.inf
    nonocc = rng.choice(np.array([255, 0, 128], np.uint8), size=(H, W), p=[0.6, 0.3, 0.1])
    return gt, nonocc


def check_render_evaluation(E, gt, nonocc, modes=(0, 1), precisions=PRECISIONS):
    """lexp_render_evaluation of the device state of each view against the oracle on that state, bit for bit; and partial requests."""
    E.set_ground_truth(gt, nonocc)
    n = 0
    for m in modes:
        lab = E.pm_get(m)[1]
        for precision, threshold in precisions:
            got = E.render_evaluation(m, precision, threshold)
            want = V.eval_images(lab, gt, nonocc, precision, threshold, E.MAX_DISPARITY)
            for k, g, w in zip("DNE", got, want):
                assert g.dtype == np.uint8 and g.shape == w.shape, k
                bad = np.argwhere(g != w)
                assert bad.size == 0, (k, m, precision, bad[:5], g[tuple(bad[0])], w[tuple(bad[0])])
            n += 1
        # one image alone: the others are not requested (NULL pointers)
        e = np.zeros((E.height, E.width), np.uint8)
        check(lib().lexp_render_evaluation(E._h, m, float(precisions[-1][0]), float(precisions[-1][1]), None, None, e.ctypes.data))
        assert np.array_equal(e, want[2])
    return n


def check_render_consistency(E):
    """lexp_render_consistency of both views' device state against the oracle, bit for bit."""
    lab0, lab1 = E.pm_get(0)[1], E.pm_get(1)[1]
    got = E.render_consistency()
    want = V.check_images(lab0, lab1, E.MIN_DISPARITY, E.MAX_DISPARITY)
    for m in range(2):
        bad = np.argwhere(got[m] != want[m])
        assert bad.size == 0, (m, bad[:5])
    return got


def set_designed_state(E, modes, seed):
    for m in modes:
        lab = designed_labeling(E.height, E.width, E.MAX_DISPARITY, seed + 17 * m)
        E.pm_begin(m, None, lab)


def expected_images(views, pm, gc):
    """(index, mode, kind) of every image FastGCStereo::run writes (Evaluator.h:164-166, FastGCStereo.h:160-167,188-195,208-215)."""
    out = []
    pts = RC.expected_indices(views, pm, gc)
    ends = {it + 1 for it in range(pm + gc)} | {pm + gc + 1}
    for j, (i, m) in enumerate(pts):
        out += [(i, m, k) for k in "DNE"]
        last_of_point = j + 1 == len(pts) or pts[j + 1][0] != i
        if len(views) == 2 and last_of_point and i in ends:
            out += [(i, 0, "C"), (i, 1, "C")]
    return out


def composed_run_images(E, views, pm, gc, units, props, seed, precision, threshold, gt=None, nonocc=None):
    """run_checks.composed_run with the images of every point rendered through lexp_render_*: [(index, mode, kind, image, oracle)] and
    view 0's final labeling.  oracle: with gt given, vis_oracle's image of the state at that point, else None."""
    sw = {m: NativePMSweep(E, unit_sizes=units, proposers=props, mode=m) for m in views}
    out = []

    def ev(i, m):
        want = [None] * 3
        if gt is not None:
            want = V.eval_images(E.pm_get(m)[1], gt, nonocc, precision, threshold, E.MAX_DISPARITY)
        for k, img, w in zip("DNE", E.render_evaluation(m, precision, threshold), want):
            out.append((i, m, k, img, w))

    def cc(i):
        if len(views) == 2:
            want = [None] * 2
            if gt is not None:
                want = V.check_images(E.pm_get(0)[1], E.pm_get(1)[1], E.MIN_DISPARITY, E.MAX_DISPARITY)
            for m, (img, w) in enumerate(zip(E.render_consistency(), want)):
                out.append((i, m, "C", img, w))
    try:
        for m in views:
            sw[m].begin()
            sw[m].random_start(run_seed(seed, m, RUN_INIT))
            ev(0, m)
        for it in range(pm):
            for m in views:
                sw[m].iteration(it, run_seed(seed, m, RUN_PM, it))
                ev(it + 1, m)
            cc(it + 1)
        for it in range(gc):
            for m in views:
                sw[m].gc_iteration(it, run_seed(seed, m, RUN_GC, it))
                ev(it + 1 + pm, m)
            cc(it + 1 + pm)
        raw = E.pm_get(0)[1]
        if len(views) == 2:
            E.post_process(1.5)
            ev(gc + 1 + pm, 0)
            ev(gc + 1 + pm, 1)
            cc(gc + 1 + pm)
        return out, E.pm_get(0)[1], raw
    finally:
        for s in sw.values():
            s.close()


def check_run_images(mk, views, pm, gc, units, props, seed, precision=0.25, threshold=0.5):
    """lexp_run_ex with an image callback on one context, lexp_run without it on a second and the composed run on a third: the images at
    exactly the reference's (index, mode, kind) list, each equal to lexp_render_* of the composed run at that point and to the oracle
    of the composed run's state there; labelings, evaluations and indices unchanged by the images."""
    Ea, Eb, Ec = mk(), mk(), mk()
    try:
        gt, nonocc = RC.synthetic_gt(Ea, seed)
        for E in (Ea, Eb, Ec):
            E.set_ground_truth(gt, nonocc)
        calls_a, calls_b, imgs = [], [], []
        order = []
        lab_a, raw_a = Ea.run(gc, views, pm, None, units, props, seed, precision, threshold,
                              callback=lambda i, m, r, t: (calls_a.append((i, m, r, t)), order.append((i, m, "eval"))),
                              image_callback=lambda i, m, k, a: (imgs.append((i, m, k, a)), order.append((i, m, k))))
        lab_b, raw_b = Eb.run(gc, views, pm, None, units, props, seed, precision, threshold, callback=lambda i, m, r, t: calls_b.append((i, m, r, t)))
        want, lab_c, raw_c = composed_run_images(Ec, views, pm, gc, units, props, seed, precision, threshold, gt, nonocc)
        assert [(i, m, k) for i, m, k, _ in imgs] == expected_images(views, pm, gc)
        assert [(i, m, k) for i, m, k, _, _ in want] == expected_images(views, pm, gc)
        # the evaluation callback comes first at every point, then D, N, E
        for j in [j for j, t in enumerate(order) if t[2] == "eval"]:
            assert [t[2] for t in order[j:j + 4]] == ["eval", "D", "N", "E"]
        for (i, m, k, g), (_, _, _, r, w) in zip(imgs, want):
            assert g.dtype == np.uint8 and g.shape == w.shape, (i, m, k)
            assert np.array_equal(g, r) and np.array_equal(g, w), (i, m, k)
        assert [(i, m, r) for i, m, r, _ in calls_a] == [(i, m, r) for i, m, r, _ in calls_b]
        for a, b in ((lab_a, lab_b), (raw_a, raw_b), (lab_a, lab_c), (raw_a, raw_c)):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        return imgs
    finally:
        Ea.close(); Eb.close(); Ec.close()


def vis_energy(H, W, D, windR, naive=False, min_disp=0.0, seed=0):
    """run_checks.scene_energy, optionally with MIN_DISPARITY != 0 (the C images' offset)."""
    if min_disp == 0.0:
        return RC.scene_energy(H, W, D, windR, naive=naive, seed=seed)
    from lexp_testlib import make_scene
    imL, imR, volL, volR = make_scene(H, W, D, seed=seed)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.CostVolumeEnergy(imL, imR, volL, volR, prm, D - 1, min_disp)
    E.set_smoothness(**RC.SMOOTH)
    return E
