"""RansacProposer on the device (LEXP_PROP_RANSAC, csrc/lexp_ransac.cuh) against oracle/ransac_oracle.py, which restates
RANSACPlane (Proposer.h:155-312) under the contract of DESIGN.md section 3f.

Proposer level: the state is set with lexp_pm_begin, one RANSAC step records its planes through d_planes_out, and the oracle fits
the same snapshot with the same random streams: the planes must be bit-identical.  Sweep level, with sweep.V3_PROPOSERS_REFERENCE:
one pm iteration with every step certified by tests/pm_step_rig.py (each RANSAC proposal bit for bit against the oracle's fit of the
device's state before the step, the update rule, the proposal costs), and one graph-cut iteration, group by group, whose RANSAC
proposals must equal the oracle's fit of the device's state and whose RANSAC moves are certified against the exact minimum cut."""
import numpy as np
import pytest

from oracle import lexp_oracle as O
from oracle import ransac_oracle as RO
from lexp_replay import certify_gc_step
from lexp_testlib import TorchDeviceMemory, energy_and_oracle, make_scene, pdl_off
from pm_step_rig import Rig, run_sweep

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def devmem():
    return TorchDeviceMemory()


def _plane_at(lab, rect, a, b, c):
    x, y, w, h = rect
    lab[y:y + h, x:x + w] = (a, b, c, 0.0)


def designed_scene(H=64, W=96, seed=3):
    """A labeling whose unit regions are the designed cases, and the units: [(rect, what)]."""
    rng = np.random.default_rng(seed)
    lab = np.zeros((H, W, 4), np.float32)
    lab[..., 2] = 20.0
    units = []

    def unit(rect, what):
        units.append((rect, what))
        return rect
    r = unit((0, 0, 20, 20), "dyadic plane + gross outliers")
    _plane_at(lab, r, 0.25, -0.125, 30.0)
    m = rng.random((20, 20)) < 0.25
    lab[0:20, 0:20][m] = np.stack([np.zeros(m.sum()), np.zeros(m.sum()), rng.uniform(0, 60, m.sum()), np.zeros(m.sum())], 1)
    r = unit((24, 0, 20, 20), "two planes split 60/40")
    _plane_at(lab, (24, 0, 12, 20), 0.5, 0.0, 2.0)
    _plane_at(lab, (36, 0, 8, 20), -0.25, 0.25, 40.0)
    r = unit((48, 0, 16, 12), "fronto-parallel")
    _plane_at(lab, r, 0.0, 0.0, 17.5)
    r = unit((68, 0, 20, 20), "random labels (low inlier ratio, many batches)")
    lab[0:20, 68:88, 0] = rng.uniform(-1, 1, (20, 20))
    lab[0:20, 68:88, 1] = rng.uniform(-1, 1, (20, 20))
    lab[0:20, 68:88, 2] = rng.uniform(0, 80, (20, 20))
    r = unit((0, 24, 30, 1), "1 x k: collinear")
    _plane_at(lab, r, 0.5, 0.0, 3.0)
    lab[24, 5:10, 2] += 7.0
    r = unit((32, 24, 1, 25), "k x 1: collinear")
    _plane_at(lab, r, 0.0, -0.5, 40.0)
    r = unit((36, 24, 1, 1), "n = 1")
    r = unit((40, 24, 3, 1), "n = 3")
    r = unit((46, 24, 2, 1), "n = 2")
    r = unit((52, 24, 12, 12), "NaN and inf labels")
    _plane_at(lab, r, 0.125, 0.125, 10.0)
    lab[24:28, 52:56, 2] = np.nan
    lab[30, 52:60, 0] = np.inf
    lab[31, 52:60, 1] = -np.inf
    r = unit((68, 24, 24, 20), "noisy slanted plane")
    X, Y = np.meshgrid(np.arange(68, 92), np.arange(24, 44))
    lab[24:44, 68:92, 0] = 0.3
    lab[24:44, 68:92, 1] = -0.2
    lab[24:44, 68:92, 2] = (30.0 - 0.3 * X + 0.2 * Y + rng.normal(0, 0.6, X.shape)).astype(np.float32)
    r = unit((0, 48, 40, 16), "every label non-finite")
    lab[48:64, 0:40, 2] = np.nan
    return lab, units


def make_energy(H, W, D, windR=8, naive=False):
    import localexpstereo_b200 as L
    imL, imR, volL, volR = make_scene(H, W, D)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    return L.CostVolumeEnergy(imL, None, volL, None, prm, D - 1)


def run_ransac_step(devmem, E, lab, units, seed, cell_ids=None, gc=False):
    """One LEXP_PROP_RANSAC step over `units` (one plan, one call per unit, targetRect = unit) from the labeling `lab`; returns the
    recorded planes [n][4]."""
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import window_rects
    H, W = lab.shape[:2]
    pl = E.make_plan(window_rects(units, E.params.windR, W, H), units)
    try:
        pl.set_units(units, cell_ids)
        E.pm_begin(0, None, lab)
        out = devmem.zeros((len(units), 4), fill=-7.0)
        E.pm_reset_sync()
        if gc:
            pl.gc_step(L.PROP_RANSAC, 0, seed, d_planes_out=devmem.ptr(out))
        else:
            pl.pm_step(0, L.PROP_RANSAC, 0, seed, d_planes_out=devmem.ptr(out))
        E.sync()
        return np.array(devmem.download(out))
    finally:
        pl.close()


def oracle_planes(lab, units, seed, cell_ids=None):
    ids = range(len(units)) if cell_ids is None else cell_ids
    return np.stack([RO.ransac_proposal(O.pm_rng_state(seed, i), lab, u)[0] for i, u in zip(ids, units)])


def check_designed_units(devmem):
    lab, cases = designed_scene()
    units = [r for r, _ in cases]
    E = make_energy(lab.shape[0], lab.shape[1], 16)
    try:
        for seed in (1, 0xDEADBEEF12345678):
            dev = run_ransac_step(devmem, E, lab, units, seed)
            ref = oracle_planes(lab, units, seed)
            bad = [cases[i][1] for i in range(len(units)) if not np.array_equal(dev[i].view(np.uint32), ref[i].view(np.uint32))]
            assert not bad, f"seed {seed}: device plane differs from the oracle in: {bad}\n{dev}\n{ref}"
            what = {w: i for i, (_, w) in enumerate(cases)}
            # the double solve recovers exact planes up to its rounding (~1e-14 in the slopes)
            assert np.allclose(dev[what["fronto-parallel"]], [0, 0, 17.5, 0], rtol=0, atol=1e-9)
            assert np.allclose(dev[what["dyadic plane + gross outliers"]], [0.25, -0.125, 30.0, 0], rtol=0, atol=0.01)   # outliers within 1 px join the refit
            for w in ("n = 1", "n = 2", "n = 3", "every label non-finite"):
                assert not dev[what[w]].any(), w
        # the graph-cut step takes the same proposals
        E.set_smoothness()
        dev_gc = run_ransac_step(devmem, E, lab, units, 1, gc=True)
        assert np.array_equal(dev_gc, oracle_planes(lab, units, 1))
    finally:
        E.close()


def test_designed_units(devmem):
    """Dyadic plane with outliers, two planes, fronto-parallel, collinear 1 x k / k x 1 units, n <= 3, NaN / inf labels, random labels."""
    check_designed_units(devmem)


def test_argument_errors():
    """LEXP_PM_INIT with RANSAC, K != 1 and world > 1 in the sweep object: LEXP_ERR_INVALID, nothing enqueued."""
    import localexpstereo_b200 as L
    from localexpstereo_b200._capi import LexpError
    from localexpstereo_b200.sweep import NativePMSweep, PMSweep
    H, W, D = 40, 56, 8
    E = make_energy(H, W, D)
    try:
        units = [(0, 0, 8, 8), (16, 0, 8, 8)]
        pl = E.make_plan(units, units)
        pl.set_units(units)
        E.pm_begin(0)
        n0 = E.launch_count
        with pytest.raises(LexpError, match="RANSAC"):
            pl.pm_step(0, L.PROP_RANSAC, 0, 1, init=True)
        assert E.launch_count == n0
        pl.close()
        for props, world, what in (([[(L.PROP_EXPANSION, 1), (L.PROP_RANSAC, 2)]], 1, "K != 1"), ([[(L.PROP_RANSAC, 1)]], 2, "world > 1")):
            with pytest.raises(LexpError, match="RANSAC"):
                NativePMSweep(E, unit_sizes=[8], proposers=props, world=world)
            with pytest.raises(ValueError, match="RANSAC"):
                PMSweep(E, unit_sizes=[8], proposers=props, world=world)
        assert E.launch_count == n0
    finally:
        E.close()


class _Recording:
    """Device memory that keeps the buffers it hands out (the planes certify_gc_step records)."""

    def __init__(self, devmem):
        self.devmem, self.made = devmem, []

    def zeros(self, shape, fill=0.0):
        t = self.devmem.zeros(shape, fill)
        self.made.append(t)
        return t

    def __getattr__(self, name):
        return getattr(self.devmem, name)


# ---- sweeps with the reference's proposer lists ------------------------------------------------------------------------
def sweep_replay(E, S, iteration, seed, devmem):
    """One graph-cut iteration of S issued group by group, with the device's state read back before every RANSAC step: each RANSAC
    proposal must equal the oracle's fit of that state, bit for bit, and every move of the step is certified with certify_gc_step.
    Returns the number of RANSAC proposals checked."""
    import localexpstereo_b200 as L
    T = dict(n_r=0, n_moves=0)

    def issue(g, steps):
        for k, kind, m, sd, _ in steps:
            if kind != L.PROP_RANSAC:
                g.plan.gc_step(kind, m, sd, mode=S.mode)
                continue
            E.sync()
            ref = oracle_planes(S.get()[1], g.units, sd, g.ids)   # the oracle's fit of the device's state right before the step
            cap = _Recording(devmem)
            T["n_moves"] += len(certify_gc_step(E, g.plan, g.targets, S.mode, 1.0, 1.0, cap, kind=kind, m=m, seed=sd, ties_ok=True))
            planes = np.array(devmem.download(cap.made[0]))
            bad = np.nonzero((planes.view(np.uint32) != ref.view(np.uint32)).any(axis=1))[0]
            assert not len(bad), f"layer {g.layer} group {g.group} step {k}: cells {bad[:5]}: device {planes[bad[:3]]} oracle {ref[bad[:3]]}"
            T["n_r"] += len(ref)

    for _ in S.walk(iteration, seed, issue):
        pass
    assert T["n_moves"] == T["n_r"]
    return T["n_r"]


def reference_list_gc_iteration(devmem, scene, units, D, windR, seed=5, naive=False):
    """One graph-cut iteration with V3_PROPOSERS_REFERENCE through sweep_replay, after one pm iteration on the cost-volume energy (as
    FastGCStereo::run does before its graph-cut loop; MiddV2 runs none)."""
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import GCSweep, V3_PROPOSERS_REFERENCE
    E, _ = energy_and_oracle(scene, D, windR, naive=naive, **(dict(th_col=0.5) if naive else {}))
    S = GCSweep(E, unit_sizes=units, proposers=V3_PROPOSERS_REFERENCE)
    try:
        labels = synth.synthetic_planes(S.init_units, 1, D, seed)[0]
        S.begin()
        S.init(labels)
        if not naive:
            S.iteration(0, seed)
        E.sync()
        return sweep_replay(E, S, 0 if naive else 1, seed, devmem)
    finally:
        S.close()
        E.close()


def reference_list_pm_iteration(devmem, scene, units, windR, seed=5):
    """The initialisation and one pm iteration with V3_PROPOSERS_REFERENCE on the cost-volume energy, every step certified by
    pm_step_rig (RANSAC proposals bit for bit).  Returns the rig's Tally."""
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import V3_PROPOSERS_REFERENCE
    imL, _, volL, _ = scene
    R = Rig(devmem, imL, None, volL, None, windR, units, V3_PROPOSERS_REFERENCE)
    try:
        labels = synth.synthetic_planes(R.S.init_units, 1, int(volL.shape[0]), seed)[0]
        return run_sweep(R, labels, 1, seed, what=f"reference lists, {R.H} x {R.W}, windR {windR}")
    finally:
        R.close()


def test_pm_and_gc_iteration_on_the_cones_crop(devmem):
    """One pm and one graph-cut iteration with the reference's lists on the cones crop (cost-volume energy), and one graph-cut
    iteration of the image-based energy (MiddV2 mode)."""
    import lexp_golden
    G = lexp_golden.load()
    scene = (G["imL"], G["imR"], G["volL"], G["volR"])
    T = reference_list_pm_iteration(devmem, scene, [6, 18, 40], G["windR"])
    assert T.ransac > 300
    for naive in (False, True):
        n_r = reference_list_gc_iteration(devmem, scene, [6, 18, 40], G["D"], G["windR"], naive=naive)
        print(f"gc naive={naive}: {n_r} RANSAC proposals bit-identical; every move certified")
        assert n_r > 300


def check_native_equals_python(with_gc=True):
    """NativePMSweep (lexp_pm_sweep_*) against PMSweep with the reference's lists: init, two pm iterations, one graph-cut iteration."""
    import localexpstereo_b200 as L
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import NativePMSweep, PMSweep, GCSweep, V3_PROPOSERS_REFERENCE
    H, W, D, windR = 64, 88, 12, 12
    imL, imR, volL, volR = make_scene(H, W, D)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    outs = []
    for cls in (GCSweep, NativePMSweep):
        E = L.CostVolumeEnergy(imL, None, volL, None, prm, D - 1)
        S = cls(E, unit_sizes=[8, 22, 40], proposers=V3_PROPOSERS_REFERENCE)
        try:
            E.set_smoothness()
            labels = synth.synthetic_planes(L.LayerManager(W, H, windR).addLayer(8).unitRegions, 1, D, 5)[0]
            S.begin(); S.init(labels)
            n = [S.iteration(it, 77) for it in (0, 1)]
            if with_gc:
                n.append(S.gc_iteration(2, 77))
            E.sync()
            outs.append((n, S.get()))
        finally:
            S.close(); E.close()
    assert outs[0][0] == outs[1][0]
    assert np.array_equal(outs[0][1][0], outs[1][1][0]) and np.array_equal(outs[0][1][1], outs[1][1][1])


def test_native_sweep_equals_python_with_reference_lists():
    check_native_equals_python()


def test_reference_lists_launch_chains_equal_serialized(side_stream):
    """The reference-list pm iteration on a caller stream, eagerly and as one captured iteration replayed, against a context whose
    launches are all serialized (LEXP_PDL_OFF=1): bit-identical states, and the chain still overlaps around the RANSAC steps."""
    import torch
    import localexpstereo_b200 as L
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import PMSweep, V3_PROPOSERS_REFERENCE
    H, W, D, windR = 291, 437, 40, 12
    imL, imR, volL, volR = make_scene(H, W, D)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    with pdl_off():
        R = L.CostVolumeEnergy(imL, None, volL, None, prm, D - 1)
    E = L.CostVolumeEnergy(imL, None, volL, None, prm, D - 1)
    its = [0, 1, 2, 2, 2]
    try:
        Sr = PMSweep(R, proposers=V3_PROPOSERS_REFERENCE)
        labels = synth.synthetic_planes(Sr.init_units, 1, D, 3)[0]
        Sr.begin(); Sr.init(labels)
        want = []
        for it in its:
            Sr.iteration(it, 99)
            want.append(Sr.get())
        assert R.overlapped_launch_count == 0
        Sr.close()
        E.set_stream(side_stream.cuda_stream)
        S = PMSweep(E, proposers=V3_PROPOSERS_REFERENCE)
        S.begin(); S.init(labels)
        g = None
        for j, it in enumerate(its):
            c0 = E.overlapped_launch_count
            if j < 2:
                n = S.iteration(it, 99)
                n_ransac = sum(1 for (li, gi, gp, _) in S.schedule if gp is not None)
                overl = E.overlapped_launch_count - c0
                # every launch may overlap its predecessor except the first of the iteration, each RANSAC step's two launches
                assert overl == n - 1 - n_ransac, (overl, n, n_ransac)
            else:
                if g is None:
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.stream(side_stream):
                        with torch.cuda.graph(g):
                            E.set_stream(torch.cuda.current_stream().cuda_stream)
                            S.iteration(it, 99)
                        E.set_stream(side_stream.cuda_stream)
                with torch.cuda.stream(side_stream):
                    g.replay()
                torch.cuda.synchronize()
            got = S.get()
            assert np.array_equal(got[0], want[j][0]) and np.array_equal(got[1], want[j][1]), f"iteration {j} differs from the serialized run"
        del g
        S.close()
    finally:
        E.close(); R.close()


@pytest.fixture(scope="module")
def side_stream():
    import torch
    return torch.cuda.Stream()


def test_every_cell_of_sampled_groups_at_2048(devmem):
    """Every cell of one group per layer at 2048 x 1536 x 256 (V3 layers 20 / 61 / 184 px: ~400 / 3 700 / 34 000 points per cell), from the
    state after init and after one pm iteration: planes bit-identical to the oracle's fit of the same state."""
    import time
    import localexpstereo_b200 as L
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import PMSweep
    W, H, D, windR = 2048, 1536, 256, 20
    imL = synth.synthetic_image(H, W, 42)
    vol = np.random.default_rng(1234).random((D, H, W), dtype=np.float32)
    E = L.CostVolumeEnergy(imL, None, vol, None, L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4), D - 1)
    del vol
    S = PMSweep(E)
    try:
        labels = synth.synthetic_planes(S.init_units, 1, D, 7)[0]
        S.begin(); S.init(labels)
        for when in ("init", "iteration"):
            if when == "iteration":
                S.iteration(0, 3)
            E.sync()
            cost, lab = S.get()
            for li, gi, every in ((0, 5, 1), (1, 6, 1), (2, 9, 1)):
                g = next(gp for (l, gr, gp, _) in S.schedule if l == li and gr == gi)
                units, ids = g.units[::every], g.ids[::every]
                t0 = time.time()
                dev = run_ransac_step(devmem, E, lab, units, 11 + li, cell_ids=ids)
                ref = oracle_planes(lab, units, 11 + li, ids)
                bad = np.nonzero((dev.view(np.uint32) != ref.view(np.uint32)).any(axis=1))[0]
                assert not len(bad), f"{when}, layer {li}: cells {bad[:5]} differ: {dev[bad[:3]]} vs {ref[bad[:3]]}"
                print(f"{when} layer {li}: {len(units)} cells bit-identical ({time.time() - t0:.1f} s)")
            E.pm_begin(0, cost, lab)
    finally:
        S.close(); E.close()


def test_layer2_group_at_4k(devmem):
    """One layer-2 group at 3840 x 2160 (345-px units, ~119 000 points per cell) on a piecewise-planar state with noise."""
    import localexpstereo_b200 as L
    from localexpstereo_b200 import synth
    W, H, D, windR = 3840, 2160, 16, 20
    imL = synth.synthetic_image(H, W, 42)
    vol = np.random.default_rng(5).random((D, H, W), dtype=np.float32)
    E = L.CostVolumeEnergy(imL, None, vol, None, L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4), D - 1)
    del vol
    try:
        lm = L.LayerManager(W, H, windR)
        l0 = lm.addLayer(int(W * 0.01))
        planes = synth.synthetic_planes(l0.unitRegions, 1, D, 9)[0]
        lab = np.zeros((H, W, 4), np.float32)
        for (x, y, w, h), p in zip(l0.unitRegions, planes):
            lab[y:y + h, x:x + w] = p
        lab[..., 2] += np.random.default_rng(2).normal(0, 0.3, (H, W)).astype(np.float32)
        l2 = lm.addLayer(int(W * 0.09))
        cells = l2.disjointRegionSets[0]
        units = [l2.unitRegions[r] for r in cells]
        assert max(u[2] * u[3] for u in units) > 110000
        dev = run_ransac_step(devmem, E, lab, units, 21, cell_ids=cells)
        ref = oracle_planes(lab, units, 21, cells)
        assert np.array_equal(dev.view(np.uint32), ref.view(np.uint32)), (dev, ref)
    finally:
        E.close()
