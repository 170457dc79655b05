"""Device-side PatchMatch phase (SURVEY.md section 8 f-1): FastGCStereo::run's pmInit iterations -- initCurrentFast, then
localExpansionMovesForLayer_CPU with doGC == false (FastGCStereo.h:22-72, 94-157) -- with proposals, unary costs and the
`mask = cur > prop; copy; setTo` update all on the device (lexp_plan_pm_step), against the numpy oracle (oracle.pm_step, which
tests/test_ref_pin.py holds bit-identical to the reference's own loop + proposers compiled in oracle/_ref).

Parity protocol (SURVEY.md 8d: "deterministic pm-phase replay"): the device sweep records the plane every (cell, step)
evaluated; the oracle replays that fixed plane sequence step by step.  Then (1) at every step the oracle's own proposer, run on
the oracle's state with the same random stream, must produce the plane the device produced; (2) the final costs agree to 1e-4 and
the final labels are identical except at pixels where the competing costs themselves agree to 1e-4 (the FP32 filter of the device
vs the reference's double filter can order two nearly equal costs differently)."""
import numpy as np
import pytest

from oracle import lexp_oracle as O
from lexp_testlib import REL_TOL, ABS_FLOOR, make_scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def devmem():
    from test_gpu_parity import _TorchDeviceMemory
    return _TorchDeviceMemory()


def run_pm_replay(devmem, H, W, D, windR, units, proposers, iterations=1, seed=1234, scene=None, mode=0):
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import PMSweep, expand_proposers
    imL, imR, volL, volR = scene if scene is not None else make_scene(H, W, D)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.CostVolumeEnergy(imL, imR if mode else None, volL, volR if mode else None, prm, D - 1)
    Or = O.CostVolumeEnergyOracle(imL, imR if mode else None, volL, volR if mode else None, windR, 1e-4, 0.5, D - 1)
    S = PMSweep(E, unit_sizes=units, proposers=proposers, mode=mode)
    try:
        # ---- device: begin (cost = +inf), initCurrentFast with seeded random labels, `iterations` pm iterations
        rng = O.CvRNG(seed)
        init_labels = np.stack([O.create_random_label(rng, u[0] + rng.uniform_int(0, u[2]), u[1] + rng.uniform_int(0, u[3]), 0.0, D - 1.0)
                                for u in S.init_units])
        S.begin()
        S.init(init_labels)
        rec, rec_host = {}, {}
        for it in range(iterations):
            for g in S.groups:
                nst = len(expand_proposers(proposers[g.layer], it, D - 1.0))
                rec[(it, g.layer, g.group)] = devmem.zeros((nst, g.plan.num_calls, 4))
            S.iteration(it, seed, planes_out={(l, gr): devmem.ptr(rec[(it, l, gr)]) for (i2, l, gr) in rec if i2 == it})
        E.sync()
        cost_d, lab_d = S.get()
        for k, v in rec.items():
            rec_host[k] = devmem.download(v)
        # ---- oracle: same initialisation, then the fixed plane sequence step by step
        cost_o = np.full((H, W), np.inf, np.float32)
        lab_o = np.zeros((H, W, 4), np.float32)
        R = windR
        fr0 = [(max(x - R, 0), max(y - R, 0), min(x + w + R, W) - max(x - R, 0), min(y + h + R, H) - max(y - R, 0)) for (x, y, w, h) in S.init_units]
        O.pm_step(Or, S.init_units, S.init_units, fr0, 0, 0, 0, None, cost_o, lab_o, planes=init_labels, init=True, mode=mode)
        r = oracle_pm_replay(Or, S, cost_o, lab_o, rec_host, range(iterations), seed, D)
        return dict(r, cost_d=cost_d, lab_d=lab_d)
    finally:
        S.close()
        E.close()


def oracle_pm_replay(Or, S, cost_o, lab_o, rec_host, iterations, seed, D):
    """The oracle half of the parity protocol: from the state (cost_o, lab_o), which it updates in place, the oracle runs the pm
    iterations `iterations` of the PMSweep S with the planes the device recorded, rec_host[(iteration, layer, group)] = [steps][n][4].
    At every step the oracle's own proposer, run on the oracle's state with the launch's random stream, is compared with the recorded
    plane.  Returns the oracle's state and the proposal counts that check_pm_result reads."""
    from localexpstereo_b200.sweep import expand_proposers, pm_seed
    n_prop = n_same = n_close = 0
    cell_base = np.cumsum([0] + [len(l.unitRegions) for l in S.lm.layers])
    for it in iterations:
        for g in S.groups:
            lay = S.lm.layers[g.layer]
            us = [lay.unitRegions[r] for r in g.cells]; ts = [lay.sharedRegions[r] for r in g.cells]; fs = [lay.filterRegions[r] for r in g.cells]
            ids = cell_base[g.layer] + g.cells
            for k, (kind, m) in enumerate(expand_proposers(S.proposers[g.layer], it, D - 1.0)):
                dev_planes = rec_host[(it, g.layer, g.group)][k]
                sd = pm_seed(seed, S.mode, it, g.layer, g.group, k)
                for i, u in enumerate(us):   # (1) the oracle's proposer on the oracle's state
                    mine = O.pm_proposal(kind, m, O.pm_rng_state(sd, ids[i]), lab_o, u, 0.0, D - 1.0)
                    n_prop += 1
                    n_same += int(np.array_equal(mine, dev_planes[i]))
                    n_close += int(np.allclose(mine, dev_planes[i], rtol=2e-6, atol=1e-6))
                O.pm_step(Or, us, ts, fs, 0, 0, 0, None, cost_o, lab_o, planes=dev_planes, mode=S.mode)
    return dict(cost_o=cost_o, lab_o=lab_o, n_prop=n_prop, n_same=n_same, n_close=n_close)


def check_pm_result(r):
    cd, co, ld, lo = r["cost_d"], r["cost_o"], r["lab_d"], r["lab_o"]
    assert np.isfinite(co).all() == np.isfinite(cd).all()
    inv = co == O.COST_FOR_INVALID
    assert np.array_equal(inv, cd == O.COST_FOR_INVALID)
    err = np.abs(cd.astype(np.float64) - co) / (REL_TOL * np.maximum(np.abs(co), ABS_FLOOR))
    assert err[~inv].max() <= 1.0, f"final cost: max err/tol {err[~inv].max():.3f}"
    diff = (ld != lo).any(axis=2)
    # a differing label is only acceptable where the two competing costs agree within the tolerance (checked above for the winner:
    # the costs are within 1e-4 of each other at such pixels) and must be rare
    assert diff.mean() < 2e-4, f"{diff.sum()} of {diff.size} labels differ"
    assert r["n_close"] == r["n_prop"], (r["n_close"], r["n_prop"])          # every proposal reproduced (FP64 sin/cos: 1e-6)
    assert r["n_same"] >= 0.98 * r["n_prop"], (r["n_same"], r["n_prop"])      # and almost all of them bit for bit
    print(f"pm replay: {r['n_prop']} proposals ({r['n_same']} bit-identical), final cost max err/tol {err[~inv].max():.3f}, "
          f"{int(diff.sum())} of {diff.size} labels differ")


def test_pm_phase_replay_small(devmem):
    """Two layers, all three proposal kinds, two pm iterations on a small scene (generic-radius kernel, R = 6)."""
    import localexpstereo_b200 as L
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 3)], [(L.PROP_EXPANSION, 2), (L.PROP_RANDOM, 1)]]
    check_pm_result(run_pm_replay(devmem, 72, 96, 12, 12, [8, 22], props, iterations=2, seed=5))


def test_pm_phase_replay_right_view(devmem):
    """mode = 1 (the right view of doDual runs, FastGCStereo.h:145-157): its own volume, guide and state."""
    import localexpstereo_b200 as L
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 1)]]
    check_pm_result(run_pm_replay(devmem, 60, 80, 10, 12, [8, 22], props, iterations=1, seed=11, mode=1))


def test_pm_phase_replay_r10(devmem):
    """The R = 10 instantiation (windR 20, the BASELINE configuration), three layers with multi-tile cells in the last one."""
    import localexpstereo_b200 as L
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 4)], [(L.PROP_EXPANSION, 2), (L.PROP_RANDOM, 1)], [(L.PROP_EXPANSION, 2), (L.PROP_RANDOM, 1)]]
    check_pm_result(run_pm_replay(devmem, 120, 170, 16, 20, [10, 31, 56], props, iterations=1, seed=9))


def test_pm_phase_full_sweep_on_the_cones_crop(devmem):
    """A full pm iteration (three layers, the reference's K = 9 / 3 / 3 evaluations per cell visit with the device schedule of
    sweep.V3_PROPOSERS_DEVICE) on the natural-image crop of data/MiddV2/cones that the golden vectors use."""
    import lexp_golden
    from localexpstereo_b200.sweep import V3_PROPOSERS_DEVICE
    G = lexp_golden.load()
    H, W = G["imL"].shape[:2]
    r = run_pm_replay(devmem, H, W, G["D"], G["windR"], [6, 18, 40], V3_PROPOSERS_DEVICE, iterations=1, seed=77,
                      scene=(G["imL"], G["imR"], G["volL"], G["volR"]))
    check_pm_result(r)
    assert r["n_prop"] > 4000


def test_pm_phase_cell_shard_two_ranks_in_one_process():
    """The multi-GPU cell shard of the PatchMatch phase with both "ranks" in this process (two contexts, lexp_pm_connect_local):
    every rank evaluates its share of the cells of every group and its kernels store accepted updates into BOTH copies of the
    state; epoch flags order the groups.  Both copies must end up bit-identical to the single-rank sweep (same cells, same random
    streams, same planes -- the shard only changes who computes what).  Ranks are issued group by group and synchronised in
    between, since two contexts on ONE device could otherwise starve each other while polling."""
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import PMSweep
    from localexpstereo_b200 import synth
    H, W, D, windR = 72, 100, 12, 12
    imL, imR, volL, volR = make_scene(H, W, D)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)], [(L.PROP_EXPANSION, 1)]]
    units = [8, 20, 36]   # the last layer has groups with a single cell: one rank sits those groups out
    Es = [L.CostVolumeEnergy(imL, None, volL, None, prm, D - 1) for _ in range(3)]
    try:
        single = PMSweep(Es[2], unit_sizes=units, proposers=props)
        labels = synth.synthetic_planes(single.init_units, 1, D, 5)[0]
        single.begin(); single.init(labels)
        for it in range(2):
            single.iteration(it, 31)
        ref_cost, ref_lab = single.get()
        ranks = [PMSweep(Es[r], unit_sizes=units, proposers=props, rank=r, world=2) for r in range(2)]
        for S in ranks:
            S.begin()
        for S in ranks:
            S.connect_local(Es[:2])
        for r, S in enumerate(ranks):
            S.init(labels[r::2])
        for E in Es[:2]:
            E.sync()
        for it in range(2):
            gens = [S.iteration_by_group(it, 31) for S in ranks]
            for _ in ranks[0].schedule:
                for g in gens:
                    next(g)
                for E in Es[:2]:
                    E.sync()
        assert any(len(o) == 1 for (_, _, _, o) in ranks[0].schedule), "the test should contain a group owned by one rank only"
        for r, S in enumerate(ranks):
            c, l = S.get()
            assert np.array_equal(c, ref_cost), f"rank {r}: currentCost differs from the single-rank sweep"
            assert np.array_equal(l, ref_lab), f"rank {r}: currentLabeling differs from the single-rank sweep"
        for S in ranks + [single]:
            S.close()
    finally:
        for E in Es:
            E.close()


def test_native_sweep_object_equals_the_python_schedule():
    """lexp_pm_sweep_* (the schedule object of the library, used by the C++ adapter) against sweep.PMSweep (one C call per proposal
    step): same launches, same seeds, same epochs -> bit-identical state, over an initialisation and two iterations including a
    RandomProposer that stops early in the second one."""
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import PMSweep, NativePMSweep
    from localexpstereo_b200 import synth
    H, W, D, windR = 64, 88, 12, 12
    imL, imR, volL, volR = make_scene(H, W, D)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 7)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]]   # 11 * 0.5^(it + i + 1) < 0.1 stops Random early
    outs = []
    launches = []
    for cls in (PMSweep, NativePMSweep):
        E = L.CostVolumeEnergy(imL, None, volL, None, prm, D - 1)
        S = cls(E, unit_sizes=[8, 22], proposers=props)
        try:
            n0 = len(S.init_units) if cls is PMSweep else S.num_init_labels
            lm = L.LayerManager(W, H, windR).addLayer(8)
            labels = synth.synthetic_planes(lm.unitRegions, 1, D, 5)[0]
            assert len(labels) == n0
            S.begin(); S.init(labels)
            launches.append([S.iteration(it, 77) for it in (0, 3)])
            outs.append(S.get())
        finally:
            S.close(); E.close()
    assert launches[0] == launches[1] and launches[0][1] < launches[0][0]
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
