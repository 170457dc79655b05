"""The contract of the device RansacProposer as oracle/ransac_oracle.py states it (DESIGN.md section 3f), checked on the CPU:
the solve against numpy's float64 least squares and OpenCV's own float cv::solve(DECOMP_SVD), computeSampleCount's edge cases, and
the sampler's triples."""
import math

import numpy as np
import pytest

from oracle import ransac_oracle as RO
from oracle import lexp_oracle as O


def _random_system(rng, n, x0, y0, size):
    xs = rng.integers(x0, x0 + size, n)
    ys = rng.integers(y0, y0 + size, n)
    b = (0.3 * xs - 0.2 * ys + 40 + rng.normal(0, 2.0, n)).astype(np.float32)
    return xs, ys, b


@pytest.mark.parametrize("n, x0, y0, size", [(3, 1500, 1000, 20), (3, 3500, 2000, 38), (400, 1500, 1000, 20), (3000, 200, 900, 184)])
def test_solve_agrees_with_float64_least_squares(n, x0, y0, size):
    """On full-rank systems the contract's solve is numpy's float64 least-squares plane: within 1e-6 px over the unit region, beyond
    the rounding of the plane's three coefficients to float that both sides apply."""
    rng = np.random.default_rng(n + x0)
    X, Y = np.meshgrid(np.arange(x0, x0 + size), np.arange(y0, y0 + size))
    worst, checked = 0.0, 0
    for _ in range(300):
        xs, ys, b = _random_system(rng, n, x0, y0, size)
        A = np.stack([xs, ys, np.ones(n)], 1).astype(np.float64)
        s = np.linalg.svd(A - [x0 + size // 2, y0 + size // 2, 0], compute_uv=False)
        if s[-1] < 1e-3 * s[0]:   # nearly collinear: the least-squares plane itself is ill-determined
            continue
        ref = np.linalg.lstsq(A, b.astype(np.float64), rcond=None)[0]
        got = RO.fit_plane(xs, ys, b, (x0 + size // 2, y0 + size // 2)).astype(np.float64)
        r32 = ref.astype(np.float32).astype(np.float64)
        plane = lambda p: p[0] * X + p[1] * Y + p[2]
        slack = np.abs(plane(r32) - plane(ref)).max() + np.abs(plane(np.spacing(np.abs(r32.astype(np.float32))).astype(np.float64)) - 0).max()
        worst = max(worst, float(np.abs(plane(got) - plane(ref)).max() - slack))
        checked += 1
    assert checked > 100 and worst <= 1e-6, (checked, worst)


def test_rank_deficient_systems_give_the_minimum_norm_solution():
    """Collinear points (1 x k and k x 1 units, repeated points): the minimum-norm solution of the uncentred rows, as numpy's lstsq."""
    for xs, ys in ((np.arange(100, 130), np.full(30, 7)), (np.full(25, 40), np.arange(300, 325)), (np.array([5, 5, 5]), np.array([9, 9, 9]))):
        b = (0.5 * xs - 0.25 * ys + 3).astype(np.float32)
        A = np.stack([xs, ys, np.ones(len(xs))], 1).astype(np.float64)
        ref = np.linalg.lstsq(A, b.astype(np.float64), rcond=None)[0]
        got = RO.fit_plane(xs, ys, b, (xs[0], ys[0]))
        assert np.allclose(got, ref, rtol=1e-5, atol=1e-7), (got, ref)


def cv2_fit(xs, ys, b, centre=None):
    """The reference's own solve: OpenCV's float cv::solve(DECOMP_SVD) on the absolute rows (x, y, 1)."""
    import cv2
    A = np.zeros((max(len(xs), 3), 3), np.float32)   # zero rows, as the reference leaves them in its refit matrix
    A[:len(xs)] = np.stack([xs, ys, np.ones(len(xs))], 1)
    bb = np.zeros((len(A), 1), np.float32)
    bb[:len(xs), 0] = b
    if not np.isfinite(bb).all():
        return np.full(3, np.nan, np.float32)
    return cv2.solve(A, bb, flags=cv2.DECOMP_SVD)[1].ravel().astype(np.float32)


def test_rank_decisions_and_planes_against_opencv():
    """cv2.solve(DECOMP_SVD) in float32 -- the reference's solve -- against the contract's solve, on triples of 20-, 38- and 184-pixel
    units at absolute coordinates around (1500, 1000).
    Full-rank triples: OpenCV drops singular values <= 2 DBL_EPSILON * sum(w), not 2 FLT_EPSILON * sum(w); where its smallest singular
    value lies below the latter it still returns the full-rank solution (it fits the three points), like the contract.  The planes
    agree within the float rounding of badly conditioned absolute coordinates: measured here, 89 % within 1e-3 px over the unit and
    97.5 % within 1e-2 px (median 1.3e-4 px).
    Exactly collinear triples: OpenCV's float SVD leaves a smallest singular value of rounding noise (~1e-7), above 2 DBL_EPSILON sum,
    so it returns a full-rank plane driven by that noise; the contract returns the minimum-norm rank-2 plane (numpy's lstsq).  This is
    the one rank decision where the two differ (every sample of a 1 x k or k x 1 unit, and collinear triples elsewhere)."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    dbl, flt = 2 * np.finfo(np.float64).eps, 2 * np.finfo(np.float32).eps
    diffs, below_flt, n_col, col_differs = [], 0, 0, 0
    for t in range(3000):
        size = (20, 38, 184)[t % 3]
        xs, ys, b = _random_system(rng, 3, 1500, 1000, size)
        if t % 15 == 0:   # exactly collinear
            ys = 1000 + (xs - 1500) // 2
            xs = 1500 + 2 * ((xs - 1500) // 2)
        A = np.stack([xs, ys, np.ones(3)], 1).astype(np.float32)
        w = cv2.SVDecomp(A)[0].ravel()
        G = [[int((xs * xs).sum()), int((xs * ys).sum()), int(xs.sum())], [int((xs * ys).sum()), int((ys * ys).sum()), int(ys.sum())],
             [int(xs.sum()), int(ys.sum()), 3]]
        N = cv2_fit(xs, ys, b)
        got = RO.fit_plane(xs, ys, b, (1500 + size // 2, 1000 + size // 2))
        if RO.gram_rank(G) < 3:
            if len(set(zip(xs.tolist(), ys.tolist()))) < 3:
                continue
            n_col += 1
            ref = np.linalg.lstsq(A.astype(np.float64), b.astype(np.float64), rcond=None)[0]
            assert np.allclose(got, ref, rtol=1e-5, atol=1e-6)
            col_differs += int(w.min() > dbl * w.sum() and not np.allclose(N, got, rtol=1e-3, atol=1e-3))
            continue
        assert (w > dbl * w.sum()).all()
        if w.min() <= flt * w.sum():
            below_flt += 1
            assert np.abs(A.astype(np.float64) @ N - b).max() < 0.05   # the full-rank fit through the three points
        X, Y = np.meshgrid(np.arange(1500, 1500 + size), np.arange(1000, 1000 + size))
        diffs.append(float(np.abs((got[0] - N[0]) * X.astype(np.float64) + (got[1] - N[1]) * Y + (got[2] - N[2])).max()))
    d = np.array(diffs)
    print(f"{len(d)} full-rank triples: {below_flt} with a singular value below 2 FLT_EPSILON sum (OpenCV keeps it); plane difference "
          f"over the unit: median {np.median(d):.2e} px, {np.mean(d <= 1e-3):.1%} <= 1e-3 px, {np.mean(d <= 1e-2):.1%} <= 1e-2 px; "
          f"{n_col} collinear triples, {col_differs} where OpenCV returns a different (noise-driven full-rank) plane")
    assert len(d) > 2500 and below_flt > 100 and n_col > 100 and col_differs > 0.9 * n_col
    assert np.mean(d <= 1e-3) >= 0.88 and np.mean(d <= 1e-2) >= 0.97


def test_float_solve_divergence_on_the_cones_crop():
    """The reference's float solve against the contract's on every layer-0 and layer-1 cell of the cones crop after one oracle pm
    iteration, with the same samples: the share of samples whose inlier count no_i differs, and the effect on the final planes and final
    inlier counts (DESIGN.md section 3f)."""
    pytest.importorskip("cv2")
    lab, layers = cones_state_after_one_pm_iteration()
    n_s = n_diff = n_cells = n_plane = 0
    dcount = []
    for li in (0, 1):
        for r, unit in enumerate(layers[li]["unit"]):
            st = O.pm_rng_state(77 + li, r)
            p1, t1 = RO.ransac_proposal(st, lab, unit)
            p2, t2 = RO.ransac_proposal(st, lab, unit, fit=cv2_fit)
            for a, b in zip(t1, t2):
                n_s += 1
                n_diff += int(a[1] != b[1])
            X, Y, d = RO.unit_snapshot(lab, unit)
            n_cells += 1
            n_plane += int(not np.array_equal(p1, p2))
            dcount.append(int(RO.inliers(p2[:3], X, Y, d).sum()) - int(RO.inliers(p1[:3], X, Y, d).sum()))
    dc = np.array(dcount)
    print(f"{n_cells} cells: no_i differs in {n_diff} of {n_s} common samples ({n_diff / max(n_s, 1):.1%}); final plane differs in "
          f"{n_plane} cells; final inliers (float - double): mean {dc.mean():+.2f}, min {dc.min()}, max {dc.max()}, "
          f"{np.mean(dc != 0):.1%} of cells differ")
    assert n_cells > 600


def cones_state_after_one_pm_iteration():
    """The cones crop's labeling after initCurrentFast with random labels and one oracle pm iteration with the device schedule's
    proposers (layers of 6 / 18 / 40 px); returns (labeling, layers)."""
    import lexp_golden
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import V3_PROPOSERS_DEVICE, expand_proposers, pm_seed
    G = lexp_golden.load()
    H, W = G["imL"].shape[:2]
    D, windR = G["D"], G["windR"]
    Or = O.CostVolumeEnergyOracle(G["imL"], None, G["volL"], None, windR, 1e-4, 0.5, D - 1)
    layers = [O.make_layer(W, H, windR, u) for u in (6, 18, 40)]
    cost = np.full((H, W), np.inf, np.float32)
    lab = np.zeros((H, W, 4), np.float32)
    units0 = layers[0]["unit"]
    labels = synth.synthetic_planes(units0, 1, D, 5)[0]
    fr0 = [(max(x - windR, 0), max(y - windR, 0), min(x + w + windR, W) - max(x - windR, 0), min(y + h + windR, H) - max(y - windR, 0))
           for (x, y, w, h) in units0]
    O.pm_step(Or, units0, units0, fr0, 0, 0, 0, None, cost, lab, planes=labels, init=True)
    base = 0
    for li, L in enumerate(layers):
        for gi, cells in enumerate(L["groups"]):
            us = [L["unit"][r] for r in cells]; ts = [L["shared"][r] for r in cells]; fs = [L["filter"][r] for r in cells]
            for k, (kind, m) in enumerate(expand_proposers(V3_PROPOSERS_DEVICE[li], 0, D - 1.0)):
                O.pm_step(Or, us, ts, fs, kind, m, pm_seed(3, 0, 0, li, gi, k), [base + r for r in cells], cost, lab)
        base += len(L["unit"])
    return lab, layers


def test_compute_sample_count_edge_cases():
    n = 400
    assert RO.compute_sample_count(n, n) == 1                       # q = 1
    assert RO.compute_sample_count(1, n) == 1 and RO.compute_sample_count(2, n) == 1   # q = 0: log(1) = 0, -inf -> INT_MIN -> 1
    assert RO.compute_sample_count(4, 119000) == 1                  # quotient beyond the int range: INT_MIN -> 1 (x86-64)
    q = (198 / 398) * (199 / 399) * (200 / 400)
    assert RO.compute_sample_count(200, 400) == int(math.log(1 - RO.CONF) / math.log(1 - q))
    assert RO.cvt_int_x86(float("nan")) == RO.INT_MIN and RO.cvt_int_x86(-2.9) == -2 and RO.cvt_int_x86(2147483648.0) == RO.INT_MIN


def test_sampler_draws_distinct_uniform_triples():
    """The first three entries of a uniform permutation: distinct, and every ordered triple equally likely (n = 5: 60 triples)."""
    rng = O.CvRNG(O.pm_rng_state(123, 4))
    counts = {}
    for _ in range(60000):
        t = RO.draw_triple(rng, 5)
        assert len(set(t)) == 3 and all(0 <= i < 5 for i in t)
        counts[t] = counts.get(t, 0) + 1
    assert len(counts) == 60
    c = np.array(list(counts.values()))
    assert abs(c.mean() - 1000) < 1e-9 and c.min() > 850 and c.max() < 1150
