"""Pins the oracle's PatchMatch phase of the image-based energy (oracle.pm_step / pm_proposal with NaiveStereoEnergyOracle: what the
device's naive pm steps are certified against) to the reference's own loop: oracle/_ref's ref_pm_group, the body of
FastGCStereo::localExpansionMovesForLayer_CPU with doGC == false (FastGCStereo.h:30-61) driving the reference's ExpansionProposer /
RandomProposer and its NaiveStereoEnergy, with cv::theRNG() started from the same per-(cell, step) states.  CPU only."""
import numpy as np
import pytest

from oracle import build_ref
from oracle import lexp_oracle as O

if not build_ref.available():
    pytest.skip("oracle/_ref is not built", allow_module_level=True)

from oracle import ref_binding as R  # noqa: E402

TOL = 1e-4


def test_naive_pm_phase_oracle_equals_the_reference_loop():
    """Two groups of two layers (windR 20, units 5 / 15), Expansion, a replayed list and Random: the proposals are bit-identical; the
    costs agree to 1e-4 relative; a label may differ only where the two competing costs agree to 1e-4 (the truncated image cost makes
    exact FP32 ties common, and the oracle's double filter rounds differently from the reference's)."""
    H, W, D, windR = 64, 84, 32, 20
    imL, imR = O.synthetic_image(H, W, 8), O.synthetic_image(H, W, 9)
    th_col, th_grad, alpha, eps = 10.0, 2.0, 0.9, 1e-4
    ref = R.RefEnergy(imL, imR, windR=windR, eps=eps, th_col=th_col, th_grad=th_grad, alpha=alpha, max_disp=D - 1.0, min_disp=0.0, kind=1)
    ora = O.NaiveStereoEnergyOracle(imL, imR, windR, eps, th_col, th_grad, alpha, D - 1.0)
    try:
        rng = O.CvRNG(21)
        units0 = O.make_layer(W, H, windR, 5)["unit"]
        labels = np.stack([O.create_random_label(rng, u[0] + rng.uniform_int(0, u[2]), u[1] + rng.uniform_int(0, u[3]), 0.0, D - 1.0) for u in units0])
        state = {who: (np.full((H, W), np.inf, np.float32), np.zeros((H, W, 4), np.float32)) for who in ("ref", "ora")}
        ref.pm_init(units0, labels, windR, *state["ref"])
        fr0 = [(max(x - windR, 0), max(y - windR, 0), min(x + w + windR, W) - max(x - windR, 0), min(y + h + windR, H) - max(y - windR, 0))
               for (x, y, w, h) in units0]
        O.pm_step(ora, units0, units0, fr0, 0, 0, 0, None, *state["ora"], planes=labels, init=True)
        assert np.array_equal(state["ref"][1], state["ora"][1])
        list_rng = O.CvRNG(77)
        n_prop = n_px = n_diff = 0
        worst = 0.0
        for li, (u, proposers) in enumerate([(5, [(1, 1), (0, 1), (2, 3)]), (15, [(1, 2), (0, 1)])]):   # Expansion, replayed list, Random
            lay = O.make_layer(W, H, windR, u)
            for gi in (0, 5):
                cells = lay["groups"][gi]
                us = [lay["unit"][r] for r in cells]; ts = [lay["shared"][r] for r in cells]; fs = [lay["filter"][r] for r in cells]
                steps = [(k, m) for k, K in proposers for m in range(K)]       # outer_iter = 1 below: Random m = 1 + iter
                seeds = [1000 * li + 10 * gi + s for s in range(len(steps))]
                states = np.array([[O.pm_rng_state(seeds[s], 100 * li + r) for s in range(len(steps))] for r in cells], dtype=np.uint64)
                lists = np.stack([[O.create_random_label(list_rng, u_[0], u_[1], 0.0, D - 1.0)] for u_ in us])   # [n][1][4]
                # both sides start the group from the reference's state, so a tie decided differently earlier does not propagate
                oc, ol = state["ref"][0].copy(), state["ref"][1].copy()
                planes_ref, nsteps = ref.pm_group(us, ts, fs, proposers, 1, states, *state["ref"], list_planes=lists)
                assert (nsteps == len(steps)).all()
                for s, (kind, it) in enumerate(steps):
                    used = O.pm_step(ora, us, ts, fs, kind, 1 + it, seeds[s], [100 * li + r for r in cells], oc, ol,
                                     planes=lists[:, 0] if kind == 0 else None)
                    assert np.array_equal(used, planes_ref[:, s]), f"layer {li} group {gi} step {s}: proposals differ"
                    n_prop += len(used)
                rc, rl = state["ref"]
                inv = rc == O.COST_FOR_INVALID
                assert np.array_equal(inv, oc == O.COST_FOR_INVALID), f"layer {li} group {gi}: COST_FOR_INVALID mask differs"
                ok = ~inv & np.isfinite(rc)
                err = np.abs(oc[ok].astype(np.float64) - rc[ok]) / np.maximum(np.abs(rc[ok]), 1e-3)
                assert err.max() <= TOL, f"layer {li} group {gi}: currentCost max rel err {err.max():.2e}"
                worst = max(worst, float(err.max()))
                diff = (ol != rl).any(axis=2)
                if diff.any():   # each side's winner costs what the other side's does, within the tolerance
                    for y, x in np.argwhere(diff):
                        a = ora.compute_unary_potential(*_pixel_rects(x, y, fs, ts), ol[y, x])[0, 0]
                        b = ora.compute_unary_potential(*_pixel_rects(x, y, fs, ts), rl[y, x])[0, 0]
                        assert abs(float(a) - float(b)) <= TOL * max(abs(float(b)), 1e-3), (li, gi, y, x, a, b)
                n_diff += int(diff.sum()); n_px += diff.size
        assert n_diff <= 1e-3 * n_px, (n_diff, n_px)
        print(f"naive pm pin: {n_prop} proposals bit-identical, cost max rel err {worst:.2e}, {n_diff} of {n_px} labels at ties")
    finally:
        ref.close()


def _pixel_rects(x, y, filts, targets):
    """(filterRect, 1 x 1 targetRect) of the group's cell whose targetRect holds pixel (x, y)."""
    for f, (tx, ty, tw, th) in zip(filts, targets):
        if tx <= x < tx + tw and ty <= y < ty + th:
            return f, (int(x), int(y), 1, 1)
    raise AssertionError(f"pixel {(x, y)} is in no targetRect of the group")
