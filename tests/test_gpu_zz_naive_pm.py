"""The PatchMatch phase of the image-based energy (NaiveStereoEnergy, BASELINE.json configs[0] `-mode MiddV2`: initCurrentFast, two pm
iterations, then the graph-cut iterations, main.cpp:21,310-312) on the device.

Per-step certification (tests/pm_step_rig.py on the scenes of tests/naive_pm_checks.py: proposals, update rule, PatchMatch = unary
instantiation, oracle costs) on the cones crop with the reference's proposer lists, at a generic radius, with v != 0 and at
2048 x 1536; the MiddV2-shaped run with the Python and the native schedule; the launch paths; the refusal on a connected cell shard.
(Sorted after the graph-cut tests and before the large-size tests.)"""
import time

import numpy as np
import pytest

import naive_pm_checks as NP
from lexp_testlib import TorchDeviceMemory, bits, pdl_off, seeded_labels

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def devmem():
    return TorchDeviceMemory()


def same_state(a, b):
    return np.array_equal(bits(a[0]), bits(b[0])) and np.array_equal(bits(a[1]), bits(b[1]))


# ---- per-step certification ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [0, 1])
def test_every_naive_pm_step_on_the_cones_crop(devmem, mode):
    NP.scene_cones(devmem, mode)


def test_every_naive_pm_step_at_a_generic_radius(devmem):
    NP.scene_generic_radius(devmem, 0)


def test_every_naive_pm_step_with_vertical_offsets(devmem):
    NP.scene_vertical_offset(devmem, 1)


# ---- the MiddV2-shaped run ------------------------------------------------------------------------------------------------------------------
def middv2_run(S, labels, seed, pm_iterations=2, gc_iterations=2):
    """begin, init, pm iterations (the data term never rises across one), graph-cut iterations; the state after each phase."""
    S.begin()
    S.init(labels)
    out = [S.get()]
    data = S.energy.energy(S.mode)[0]
    for it in range(pm_iterations):
        S.iteration(it, seed)
        out.append(S.get())
        d = S.energy.energy(S.mode)[0]
        assert d <= data, f"pm iteration {it}: data term rose from {data!r} to {d!r}"
        assert d < data or it > 0, "the first pm iteration changed nothing"
        data = d
    for it in range(gc_iterations):
        S.gc_iteration(it, seed + 1)
        out.append(S.get())
    return out


def test_middv2_run_python_and_native_schedules_agree():
    """init, 2 pm iterations and 2 graph-cut iterations at lambda 20 on the cones crop with the reference's lists: GCSweep and the
    library's own schedule object (NativePMSweep, what PatchMatchPhase calls) give the same bits after every phase, and a second run
    with the same seed repeats them."""
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import GCSweep, NativePMSweep
    imL, imR = NP.cones()
    D, props = 64, NP.reference_lists(3)
    smooth = dict(lam=NP.MIDDV2_LAMBDA, omega=10.0, th_smooth=1.0, epsilon=0.01)
    mk = lambda: L.NaiveStereoEnergy(imL, imR, NP.middv2_params(), D - 1)
    Ea, Eb, Ec = mk(), mk(), mk()
    try:
        A = GCSweep(Ea, unit_sizes=NP.MIDDV2_UNITS, proposers=props, **smooth)
        C = GCSweep(Ec, unit_sizes=NP.MIDDV2_UNITS, proposers=props, **smooth)
        Eb.set_smoothness(**smooth)
        B = NativePMSweep(Eb, unit_sizes=NP.MIDDV2_UNITS, proposers=props)
        labels = seeded_labels(A, 12)
        assert B.num_init_labels == len(labels)
        t0 = time.perf_counter()
        ra = middv2_run(A, labels, 2024)
        t1 = time.perf_counter()
        rb = middv2_run(B, labels, 2024)
        rc = middv2_run(C, labels, 2024)
        for i, (a, b, c) in enumerate(zip(ra, rb, rc)):
            assert same_state(a, b), f"phase {i}: NativePMSweep differs from GCSweep"
            assert same_state(a, c), f"phase {i}: a second run with the same seed differs"
        assert not same_state(ra[1], ra[0]) and not same_state(ra[3], ra[2])
        print(f"MiddV2-shaped run on {Ea.height} x {Ea.width}: {t1 - t0:.2f} s (Python schedule, with read-backs)")
        for S in (A, B, C):
            S.close()
    finally:
        for E in (Ea, Eb, Ec):
            E.close()


# ---- launch paths ---------------------------------------------------------------------------------------------------------------------------
PM_PREFIX, PM_REPLAYS, PM_SEED = 2, 2, 515


def test_naive_pm_launch_paths_equal_serialized():
    """PMSweep on the image-based energy: eagerly on the context's stream (overlapped launches), eagerly on a caller's stream, and
    one iteration captured into a CUDA graph and replayed -- after init and after every iteration the state equals the PDL-off
    context's, bit for bit."""
    import torch
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import PMSweep
    imL, imR = NP.cones()
    D = 64
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 3)], [(L.PROP_EXPANSION, 2)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]]
    mk = lambda: L.NaiveStereoEnergy(imL, imR, NP.middv2_params(), D - 1)
    its = list(range(PM_PREFIX)) + [PM_PREFIX] * PM_REPLAYS
    with pdl_off():
        Er = mk()
    Sr = PMSweep(Er, unit_sizes=NP.MIDDV2_UNITS, proposers=props)
    labels = seeded_labels(Sr, 5)
    Sr.begin(); Sr.init(labels)
    want = [Sr.get()]
    for it in its:
        Sr.iteration(it, PM_SEED)
        want.append(Sr.get())
    assert Er.overlapped_launch_count == 0
    Sr.close(); Er.close()
    side = torch.cuda.Stream()
    for name in ("eager", "caller stream", "graph"):
        E = mk()
        S = PMSweep(E, unit_sizes=NP.MIDDV2_UNITS, proposers=props)
        try:
            if name != "eager":
                E.set_stream(side.cuda_stream)
            S.begin(); S.init(labels)
            assert same_state(S.get(), want[0]), f"{name}: init"
            g = None
            for j, it in enumerate(its):
                if name != "graph" or j < PM_PREFIX:
                    S.iteration(it, PM_SEED)
                else:
                    if g is None:
                        g = torch.cuda.CUDAGraph()
                        with torch.cuda.stream(side):
                            with torch.cuda.graph(g):
                                E.set_stream(torch.cuda.current_stream().cuda_stream)
                                assert S.iteration(it, PM_SEED) > 0
                            E.set_stream(side.cuda_stream)
                    with torch.cuda.stream(side):
                        g.replay()
                    torch.cuda.synchronize()
                assert same_state(S.get(), want[j + 1]), f"{name}: iteration {j} (index {it})"
            assert E.overlapped_launch_count > 0, f"{name}: no launch overlapped its predecessor"
            del g
        finally:
            S.close()
            E.close()


# ---- errors ---------------------------------------------------------------------------------------------------------------------------------
def test_naive_pm_step_on_a_connected_shard_is_refused():
    """A view of the image-based energy connected to a peer (world 2) refuses a pm step with LEXP_ERR_INVALID and enqueues nothing."""
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import PMSweep
    imL, imR = NP.cones(64, 80)
    E0, E1 = (L.NaiveStereoEnergy(imL, imR, NP.middv2_params(), 31.0) for _ in range(2))
    S = PMSweep(E0, unit_sizes=[5, 15], proposers=[[(L.PROP_EXPANSION, 1)], [(L.PROP_EXPANSION, 1)]])
    try:
        S.begin(); S.init(seeded_labels(S, 3))
        E1.pm_begin(0)
        before = S.get()
        E0.pm_connect_local(0, [E0, E1])
        E1.pm_connect_local(1, [E0, E1])
        n0 = E0.launch_count
        g = S.groups[0]
        for kind, planes in ((L.PROP_EXPANSION, None), (L.PROP_LIST, np.tile(np.float32([0, 0, 3, 0]), (g.plan.num_calls, 1)))):
            with pytest.raises(L.LexpError, match="one GPU"):
                g.plan.pm_step(0, kind, 0, 1, planes=planes)
        assert E0.launch_count == n0
        E0.sync()
        assert same_state(S.get(), before)
    finally:
        S.close()
        E0.close(); E1.close()


# ---- size -----------------------------------------------------------------------------------------------------------------------------------
def test_naive_pm_iteration_at_2048x1536():
    """One pm iteration of the image-based energy at 2048 x 1536 x 256, windR 20, MiddV2's layers and the reference's lists, with
    the first and the last group of every layer certified step by step (oracle costs on sampled cells); pm_get raises on an error flag."""
    from localexpstereo_b200 import synth
    W, H, D = 2048, 1536, 256
    imL, imR = synth.synthetic_image(H, W, 42), synth.synthetic_image(H, W, 43)
    dm = TorchDeviceMemory()
    R = NP.naive_rig(dm, imL, imR, D, 20, NP.MIDDV2_UNITS, NP.reference_lists(3), q_cells=3, seed=4)
    try:
        last = {}
        for (li, gi, g, _) in R.S.schedule:
            last[li] = gi
        labels = synth.synthetic_planes(list(R.S.lm.layers[0].unitRegions), 1, D, 99)[0]
        t0 = time.perf_counter()
        R.Sq.begin()
        R.S.begin()
        R.S.init(labels)
        n, _ = R.iteration(0, 4321, certify=lambda g: g.group in (0, last[g.layer]))
        c, l = R.S.get()
        assert np.isfinite(c).all()
        print(R.T.line("2048 x 1536 x 256") + f"; {n} launches, {time.perf_counter() - t0:.1f} s in all")
        assert R.T.steps == 2 * (9 + 3 + 3)
    finally:
        R.close()
