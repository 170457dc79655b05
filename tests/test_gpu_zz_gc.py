"""(Sorted after the unary / PatchMatch / drop-in tests in the -m gpu suite: the graph-cut kernels were reworked -- shared per-node steps,
proposed heights -- after their last run on hardware.)

Pairwise terms and the expansion move on the device (SURVEY.md section 8 f-2 / f-3): StereoEnergy::initSmoothnessCoeff,
computeSmoothnessTermsExpansion (StereoEnergy.h:131-163, 398-453) and FastGCStereo::expansionMoveBK inside the graph-cut
iterations of FastGCStereo::run (FastGCStereo.h:22-72 with doGC == true, 411-597), against the numpy / C oracle
(oracle.smoothness_coeff, smoothness_terms_expansion, expansion_graph, gc_step) -- which tests/test_ref_pin.py holds against the
reference's own StereoEnergy and FastGCStereo::expansionMoveBK compiled in oracle/_ref.

Parity protocol of the moves (the same replay as the PatchMatch phase, tests/lexp_replay.py): the device sweep records the plane
and the minimum-cut energy of every (cell, step); the oracle replays that plane sequence on its own state.  Then (1) the oracle's
proposer reproduces every device proposal, (2) every move's minimum-cut energy agrees to 1e-5 (the graph the device built from ITS
unary costs and the cut it found have the value of the oracle's), (3) final costs agree to 1e-4 and final labels are identical
except for a small fraction of pixels (a cut through a tie -- the FP32 guided filter of the device against the reference's double
one -- can flip connected pixels), (4) the total energy (data + smoothness) of the two final states agrees to 1e-5."""
import numpy as np
import pytest

from oracle import lexp_oracle as O
from lexp_replay import SMOOTH, check_gc_result, oracle_init, run_gc_replay
from lexp_testlib import ABS_FLOOR, REL_TOL, TorchDeviceMemory, energy_and_oracle, make_scene, seeded_labels

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def devmem():
    return TorchDeviceMemory()


def test_smoothness_coefficients_equal_the_oracle():
    """lexp_get_smooth_coeff = initSmoothnessCoeff: max(epsilon, exp(-sum|dI| / omega)), zero towards pixels outside the image."""
    import localexpstereo_b200 as L
    H, W, D = 50, 70, 8
    imL, imR, volL, volR = make_scene(H, W, D, seed=3)
    E = L.CostVolumeEnergy(imL, imR, volL, volR, L.Parameters(windR=8, filterName="GF", filter_param1=1e-4, th_col=0.5), D - 1)
    try:
        for mode, im in ((0, imL), (1, imR)):
            for omega, eps in ((10.0, 0.01), (3.0, 0.2)):
                E.set_smoothness(1.0, omega, 1.0, eps)
                got, want = E.smooth_coeff(mode), O.smoothness_coeff(im, omega, eps)
                assert np.array_equal(got == 0, want == 0)
                assert np.allclose(got, want, rtol=2e-6, atol=0), np.abs(got - want).max()
                assert (got[want != 0] >= np.float32(eps)).all()
    finally:
        E.close()


def test_pairwise_terms_equal_the_oracle_bit_for_bit():
    """lexp_pairwise_terms = computeSmoothnessTermsExpansion(.., onlyForward = true): every product and sum is rounded separately
    on the device as in the reference, so with the device's own coefficient maps the three maps are bit-identical -- including the
    regions that touch the image border (zero margin of labeling_m / coordinates_m)."""
    import localexpstereo_b200 as L
    H, W, D = 46, 64, 10
    imL, imR, volL, volR = make_scene(H, W, D, seed=8)
    E = L.CostVolumeEnergy(imL, imR, volL, volR, L.Parameters(windR=8, filterName="GF", filter_param1=1e-4, th_col=0.5), D - 1)
    try:
        E.set_smoothness(0.7, 8.0, 0.9, 0.02)
        rng = O.CvRNG(4)
        lab = np.zeros((H, W, 4), np.float32)
        for y in range(0, H, 4):       # piecewise-constant random labels (4 x 4 blocks) with a few outliers
            for x in range(0, W, 4):
                lab[y:y + 4, x:x + 4] = O.create_random_label(rng, x, y, 0.0, D - 1.0)
        lab[5, 7] = (0.3, -0.2, 4.0, 0.0); lab[H - 1, W - 1] = (0.0, 0.0, 2.5, 0.0)
        for mode in (0, 1):
            E.pm_begin(mode, np.zeros((H, W), np.float32), lab)
            coeff = E.smooth_coeff(mode)
            regions = [(8, 6, 20, 18), (0, 0, 17, 13), (W - 9, H - 11, 9, 11), (0, 0, W, H), (30, 0, 1, 1)]
            planes = [O.create_random_label(rng, r[0], r[1], 0.0, D - 1.0) for r in regions]
            got = E.computeSmoothnessTermsExpansion(regions, planes, mode)
            for r, pl, g in zip(regions, planes, got):
                want = O.smoothness_terms_expansion(lab, pl, r, coeff, 0.7, 0.9)
                for t in range(3):
                    for fi, k in enumerate(O.FORWARD):
                        assert np.array_equal(g[t][fi], want[t][k]), (mode, r, t, k, np.abs(g[t][fi] - want[t][k]).max())
    finally:
        E.close()


def test_gc_replay_small(devmem):
    """One pm iteration, then two graph-cut iterations over two layers with all three proposal kinds (generic-radius kernel)."""
    import localexpstereo_b200 as L
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 2), (L.PROP_RANDOM, 1)]]
    check_gc_result(run_gc_replay(devmem, 72, 96, 12, 12, [8, 22], props, pm_iterations=1, gc_iterations=2, seed=5))


def test_gc_replay_right_view_strong_smoothness(devmem):
    """mode = 1 and a large lambda (the pairwise terms dominate: long chains of saturated arcs, many relabelling rounds)."""
    import localexpstereo_b200 as L
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)], [(L.PROP_EXPANSION, 1)]]
    check_gc_result(run_gc_replay(devmem, 60, 80, 10, 12, [8, 22], props, pm_iterations=0, gc_iterations=1, seed=11, mode=1,
                                  smooth=dict(lam=5.0, omega=4.0, th_smooth=1.5, epsilon=0.05)))


def test_gc_moves_never_raise_the_energy(devmem):
    """Property of an expansion move (holds for any exact minimum cut): data + smoothness energy never increases from step to step."""
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import GCSweep
    H, W, D, windR = 64, 88, 12, 12
    imL, imR, volL, volR = make_scene(H, W, D, seed=31)
    E = L.CostVolumeEnergy(imL, None, volL, None, L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5), D - 1)
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]]
    S = GCSweep(E, unit_sizes=[8, 24], proposers=props, **SMOOTH)
    coeff = O.smoothness_coeff(imL, SMOOTH["omega"], SMOOTH["epsilon"])
    try:
        rng = O.CvRNG(2)
        S.begin()
        S.init(np.stack([O.create_random_label(rng, u[0], u[1], 0.0, D - 1.0) for u in S.init_units]))
        prev = None
        for it in range(3):
            S.gc_iteration(it, 77)
            cost, lab = S.get()
            e = float(cost.astype(np.float64).sum()) + O.smoothness_cost(lab, coeff, SMOOTH["lam"], SMOOTH["th_smooth"])
            data_d, smooth_d = E.energy()      # lexp_energy: the same two sums on the device (computeSmoothnessCost, StereoEnergy.h:165-199)
            assert abs(data_d - float(cost.astype(np.float64).sum())) <= 1e-9 * abs(data_d)
            assert abs(smooth_d - O.smoothness_cost(lab, coeff, SMOOTH["lam"], SMOOTH["th_smooth"])) <= 1e-6 * max(abs(smooth_d), 1e-9)
            assert prev is None or e <= prev * (1 + 1e-6), (it, e, prev)
            prev = e
    finally:
        S.close()
        E.close()


def test_gc_replay_r10_larger_cells(devmem):
    """The R = 10 instantiation (windR 20) with three layers: cells of 30 x 30, 93 x 93 and 168 x 168 nodes (28 000 nodes in one CTA, 27
    per thread): many relabelling rounds and long residual paths."""
    import localexpstereo_b200 as L
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]]
    check_gc_result(run_gc_replay(devmem, 200, 260, 16, 20, [10, 31, 56], props, pm_iterations=1, gc_iterations=1, seed=9))


def test_gc_replay_on_the_cones_crop(devmem):
    """A pm iteration and a graph-cut iteration on the natural-image crop of data/MiddV2/cones that the golden vectors use (real
    edges in the smoothness coefficients: values from epsilon to 1 next to each other)."""
    import lexp_golden
    import localexpstereo_b200 as L
    G = lexp_golden.load()
    H, W = G["imL"].shape[:2]
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 2)], [(L.PROP_EXPANSION, 1)]]
    r = run_gc_replay(devmem, H, W, G["D"], G["windR"], [6, 18, 40], props, pm_iterations=1, gc_iterations=1, seed=77,
                      scene=(G["imL"], G["imR"], G["volL"], G["volR"]), smooth=dict(lam=1.0, omega=10.0, th_smooth=1.0, epsilon=0.01))
    check_gc_result(r)
    assert r["n_moves"] > 1000


def test_gc_iteration_on_the_image_based_energy(devmem):
    """BASELINE.json configs[0] (`-mode MiddV2`): FastGCStereo with NaiveStereoEnergy -- the reference's own demo -- whose iterations are
    all graph-cut iterations (lambda = 20, layers 5 / 15: main.cpp:72,304-305).  Entirely on the device: initCurrentFast as a unary launch +
    assignment (lexp_plan_init_step: this energy has no PatchMatch-phase kernel), then a graph-cut iteration with device-side proposals
    on the image-based unary term.
    With the truncated image-based cost many proposals evaluate to EXACTLY the current cost in the oracle (both planes leave the valid
    range: same clamped samples); the minimum cut then takes the proposal (BK's free nodes count as SOURCE) while the device's FP32
    filter separates the two costs by 1e-5 relative and keeps the current label -- same energy, another label, and a different graph for
    every later move.  So here every proposal step is checked ON ITS OWN: the oracle starts each step from the device's state before
    the step (downloaded), evaluates the device's planes, and must arrive at the device's state after the step -- minimum-cut energies
    to 1e-5, costs wherever the labels agree, labels up to those ties."""
    import lexp_golden
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import GCSweep
    G = lexp_golden.load()
    imL, imR = G["imL"], G["imR"]
    H, W = imL.shape[:2]
    D, windR = 64, 20
    lam, omega, th, eps = 20.0, 10.0, 1.0, 0.01
    E, Or = energy_and_oracle((imL, imR, None, None), D, windR, naive=True, lambda_=lam)
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)], [(L.PROP_EXPANSION, 1)]]
    S = GCSweep(E, unit_sizes=[5, 15], proposers=props, lam=lam, omega=omega, th_smooth=th, epsilon=eps)
    coeff = O.smoothness_coeff(imL, omega, eps)
    try:
        labels = seeded_labels(S, 8)
        S.begin()
        S.init(labels)
        cost_d, lab_d = S.get()
        cost_o, lab_o = oracle_init(Or, S, labels)
        assert np.array_equal(lab_d, lab_o) and np.array_equal(cost_d == O.COST_FOR_INVALID, cost_o == O.COST_FOR_INVALID)
        ok = cost_o != O.COST_FOR_INVALID
        assert (np.abs(cost_d[ok] - cost_o[ok]) <= REL_TOL * np.maximum(np.abs(cost_o[ok]), ABS_FLOOR)).all()
        n_moves = n_diff = 0
        worst_flow = worst_cost = 0.0
        for g in S.groups:
            if g.group not in (0, 5, len(S.lm.layers[g.layer].disjointRegionSets) - 1):   # three groups per layer (emulation time)
                continue
            for k, kind, m, sd in S.group_steps(g.layer, g.group, 0, 3):
                pre_c, pre_l = S.get()
                rec, flw = devmem.zeros((g.plan.num_calls, 4)), devmem.zeros((g.plan.num_calls, 2))
                g.plan.gc_step(kind, m, sd, d_planes_out=devmem.ptr(rec), d_flows_out=devmem.ptr(flw))
                E.sync()
                post_c, post_l = S.get()
                dev_planes = devmem.download(rec)
                flows_d = np.ascontiguousarray(devmem.download(flw)).view(np.float64)[:, 0]
                for i, u in enumerate(g.units):   # the device's proposer against the oracle's, on the same state
                    mine = O.pm_proposal(kind, m, O.pm_rng_state(sd, g.ids[i]), pre_l, u, 0.0, D - 1.0)
                    assert np.allclose(mine, dev_planes[i], rtol=2e-6, atol=1e-6)
                oc, ol = pre_c.copy(), pre_l.copy()
                _, flows_o = O.gc_step(Or, g.units, g.targets, g.filters, 0, 0, 0, None, oc, ol, coeff, lam, th, planes=dev_planes)
                worst_flow = max(worst_flow, float((np.abs(flows_d - flows_o) / np.maximum(np.abs(flows_o), 1e-3)).max()))
                diff = (post_l != ol).any(axis=2)
                same = ~diff & (oc != O.COST_FOR_INVALID)
                assert np.array_equal((post_c == O.COST_FOR_INVALID)[~diff], (oc == O.COST_FOR_INVALID)[~diff])
                worst_cost = max(worst_cost, float((np.abs(post_c[same].astype(np.float64) - oc[same]) / (REL_TOL * np.maximum(np.abs(oc[same]), ABS_FLOOR))).max()))
                n_diff += int(diff.sum()); n_moves += len(g.units)
        print(f"naive gc: {n_moves} moves, min-cut energy max rel err {worst_flow:.1e}, cost max err/tol {worst_cost:.3f}, {n_diff} label ties")
        assert n_moves > 300 and worst_flow <= 1e-5 and worst_cost <= 1.0, (n_moves, worst_flow, worst_cost)
        assert n_diff <= 2e-2 * H * W, n_diff
    finally:
        S.close()
        E.close()


@pytest.mark.parametrize("naive", [False, True])
def test_native_sweep_object_runs_the_same_graph_cut_iteration(naive):
    """lexp_pm_sweep_init / lexp_pm_sweep_gc_iteration (what CudaCostVolumeEnergy::PatchMatchPhase::init / graphCutIteration call) against
    the Python schedule (sweep.GCSweep): same seeds, same launches -- bit-identical state.  For the image-based energy the native init
    takes the unary launch + assignment form (lexp_plan_init_step)."""
    import lexp_golden
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import GCSweep, NativePMSweep
    G = lexp_golden.load()
    if naive:
        imL, imR, D, windR = G["imL"][:56, :72], G["imR"][:56, :72], 24, 20
        mk = lambda: L.NaiveStereoEnergy(imL, imR, L.Parameters(lambda_=20, windR=windR, filterName="GF", filter_param1=1e-4), D - 1)
        units, smooth = [5, 15], dict(lam=20.0, omega=10.0, th_smooth=1.0, epsilon=0.01)
    else:
        H, W, D, windR = 64, 88, 12, 12
        imL, _, volL, _ = make_scene(H, W, D, seed=2)
        mk = lambda: L.CostVolumeEnergy(imL, None, volL, None, L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5), D - 1)
        units, smooth = [8, 22], SMOOTH
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)], [(L.PROP_EXPANSION, 1)]]
    Ea, Eb = mk(), mk()
    try:
        A = GCSweep(Ea, unit_sizes=units, proposers=props, **smooth)
        Eb.set_smoothness(**smooth)
        B = NativePMSweep(Eb, unit_sizes=units, proposers=props)
        rng = O.CvRNG(6)
        labels = np.stack([O.create_random_label(rng, u[0], u[1], 0.0, D - 1.0) for u in A.init_units])
        assert B.num_init_labels == len(labels)
        A.begin(); B.begin()
        A.init(labels); B.init(labels)
        ca, la = A.get(); cb, lb = B.get()
        assert np.array_equal(ca, cb) and np.array_equal(la, lb)
        assert A.gc_iteration(0, 99) == B.gc_iteration(0, 99)
        ca, la = A.get(); cb, lb = B.get()
        assert np.array_equal(ca, cb) and np.array_equal(la, lb) and not np.array_equal(la[..., 2], labels[0][2] * np.ones_like(la[..., 2]))
        A.close(); B.close()
    finally:
        Ea.close(); Eb.close()
