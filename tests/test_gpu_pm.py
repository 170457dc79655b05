"""Device-side PatchMatch phase (SURVEY.md section 8 f-1): FastGCStereo::run's pmInit iterations -- initCurrentFast, then
localExpansionMovesForLayer_CPU with doGC == false (FastGCStereo.h:22-72, 94-157) -- with proposals, unary costs and the
`mask = cur > prop; copy; setTo` update all on the device (lexp_plan_pm_step), against the numpy oracle (oracle.pm_step, which
tests/test_ref_pin.py holds bit-identical to the reference's own loop + proposers compiled in oracle/_ref).

Parity protocol (SURVEY.md 8d: "deterministic pm-phase replay", tests/lexp_replay.py): the device sweep records the plane every
(cell, step) evaluated; the oracle replays that fixed plane sequence step by step.  Then (1) at every step the oracle's own proposer, run on
the oracle's state with the same random stream, must produce the plane the device produced; (2) the final costs agree to 1e-4 and
the final labels are identical except at pixels where the competing costs themselves agree to 1e-4 (the FP32 filter of the device
vs the reference's double filter can order two nearly equal costs differently)."""
import numpy as np
import pytest

from lexp_replay import check_pm_result, run_pm_replay
from lexp_testlib import TorchDeviceMemory, make_scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def devmem():
    return TorchDeviceMemory()


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
