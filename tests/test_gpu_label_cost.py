"""lexp_pm_init_from_labeling on the H100: initCurrentFast started from a given labeling (FastGCStereo.h:116-130), i.e. for every pixel
p, currentCost_(p) = ComputeUnaryPotential(F(p), {p}, ., currentLabeling_(p)) with F(p) = (p - windR, 2 windR + 1) & image.

  * designed scenes, every pixel against the C oracle and the compiled reference's own branch (ref_pm_init, one 1x1 unit per
    pixel): independent random planes beyond both ends of [MIN, MAX] with NaN / inf planes, the generic sampler, windR 20, 21, 12
    and 32, ragged widths, images smaller than the window, both views, and the image-based energy with v != 0;
  * 2048 x 1536 x 256 at windR 20: every pixel of the four 2 windR border bands plus random interior pixels (over 200 000) against
    the C oracle, and the cross-check with the initialisation of the sweep: a label painted over each layer-0 unit gives the costs
    lexp_pm_sweep_init computes (windR >= 2R: every window a pixel's cost reads lies inside its unit's filterRect too);
  * state handling: labeling unchanged, two calls / eager / caller stream / CUDA-graph replay bit-identical, a PatchMatch iteration
    right after the call, costs recomputed after lexp_post_process with lexp_energy's data term, the two-rank cell shard, errors."""
import numpy as np
import pytest

import label_cost_checks as LC
from lexp_testlib import bits, make_scene, seeded_labels
from oracle import lexp_oracle as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("windR,mode", [(20, 0), (20, 1), (21, 0), (12, 1), (32, 0)])
def test_random_planes_every_pixel(windR, mode):
    """R = 10 / 16 / generic, both views; 83 x 117: a width that is not a multiple of 4."""
    LC.check_cost_volume_scene(83, 117, 24, windR, mode=mode, seed=windR)


def test_generic_sampler_min_max():
    LC.check_cost_volume_scene(61, 90, 32, 20, MIN=3.0, MAX=27.5, seed=5)


@pytest.mark.parametrize("H,W", [(9, 80), (80, 9), (1, 61), (61, 1), (30, 30)])
def test_images_smaller_than_the_window(H, W):
    LC.check_cost_volume_scene(H, W, 16, 20, seed=H * W, nonfinite=0.01)


@pytest.mark.parametrize("mode", [0, 1])
def test_naive_energy(mode):
    """The image-based energy: each pixel's warp from its own F(p), planes with v != 0, against the numpy oracle and the reference."""
    LC.check_naive_scene(37, 51, 16, 12, mode=mode, seed=3)


def test_argument_errors():
    LC.check_argument_errors()


# ---- at the benchmark's size ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def big():
    import torch
    import localexpstereo_b200 as L
    from localexpstereo_b200 import synth
    W, H, D, windR = 2048, 1536, 256, 20
    imL = synth.synthetic_image(H, W, 42)
    vol = torch.rand((D, H, W), generator=torch.Generator(device="cuda").manual_seed(1234), device="cuda", dtype=torch.float32)
    torch.cuda.synchronize()
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.CostVolumeEnergy(imL, None, vol, None, prm, D - 1)
    vol_host = vol.cpu().numpy()
    del vol
    yield E, imL, vol_host, windR
    E.close()


def test_2048x1536_sampled_against_the_c_oracle(big):
    E, imL, vol, windR = big
    H, W = E.height, E.width
    lab = LC.random_plane_field(H, W, 0.0, 255.0, 7, nonfinite=0.001)
    got = LC.device_costs(E, lab)
    band = np.zeros((H, W), bool)
    b = 2 * windR
    band[:b] = band[-b:] = True
    band[:, :b] = band[:, -b:] = True
    rng = np.random.default_rng(3)
    inner = np.flatnonzero(~band.ravel())
    pick = np.zeros(H * W, bool)
    pick[np.flatnonzero(band.ravel())] = True
    pick[rng.choice(inner, 60000, replace=False)] = True
    ys, xs = np.divmod(np.flatnonzero(pick), W)
    assert len(ys) >= 200000
    ref = LC.c_oracle_costs(imL, vol, windR, lab, ys, xs, nthreads=32)
    worst = LC.compare(got[ys, xs], ref, "2048x1536")
    print(f"\n{len(ys)} pixels, worst err {worst:.2e}, {np.mean(ref == O.COST_FOR_INVALID):.3f} invalid")


def test_2048x1536_equals_the_sweep_initialisation(big):
    """A label painted over each layer-0 unit: the call equals lexp_pm_sweep_init with those labels, within the tolerance."""
    from localexpstereo_b200.sweep import PMSweep
    E = big[0]
    S = PMSweep(E)
    try:
        S.begin()
        S.init(seeded_labels(S, 99))
        want, lab = E.pm_get()
        got = LC.device_costs(E, lab)
        worst = LC.compare(got, want, "sweep init")
        print(f"\nagainst lexp_pm_sweep_init: worst err {worst:.2e}")
    finally:
        S.close()


def test_naive_energy_against_the_sweep_initialisation():
    """For the image-based energy the two differ: the initialisation warps over the unit's filterRect, the reference's branch over
    each pixel's own F(p).  The measured difference is printed; the invalid patterns are the same."""
    from lexp_testlib import energy_and_oracle
    from localexpstereo_b200.sweep import GCSweep
    H, W, D, windR = 240, 320, 48, 20
    E, _ = energy_and_oracle(make_scene(H, W, D, 4), D, windR, naive=True)
    S = GCSweep(E)
    try:
        S.begin()
        S.init(seeded_labels(S, 5))
        want, lab = E.pm_get()
        got = LC.device_costs(E, lab)
        inv = want == O.COST_FOR_INVALID
        assert np.array_equal(inv, got == O.COST_FOR_INVALID)
        rel = np.abs(got[~inv].astype(np.float64) - want[~inv]) / np.maximum(np.abs(want[~inv]), 1e-3)
        print(f"\nnaive energy vs its sweep initialisation: max rel diff {rel.max():.3e}, {np.mean(rel > 1e-4):.4f} of pixels beyond 1e-4")
    finally:
        S.close()
        E.close()


# ---- state handling -------------------------------------------------------------------------------------------------------------------
def _scene_energy(H=96, W=130, D=32, windR=20, seed=11, imR=True):
    import localexpstereo_b200 as L
    imL, imR_, volL, volR = make_scene(H, W, D, seed)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    return L.CostVolumeEnergy(imL, imR_ if imR else None, volL, volR if imR else None, prm, D - 1), (imL, imR_, volL, volR)


def test_eager_caller_stream_and_graph_replay_are_identical():
    import torch
    E, _ = _scene_energy()
    try:
        lab = LC.random_plane_field(E.height, E.width, 0.0, 31.0, 1)
        eager = LC.device_costs(E, lab)
        s = torch.cuda.Stream()
        E.set_stream(s.cuda_stream)
        on_stream = LC.device_costs(E, lab)
        E.pm_begin(0, cost=np.zeros((E.height, E.width), np.float32), labeling=lab)
        n0 = E.launch_count
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            E.pm_init_from_labeling(0)
        assert E.launch_count == n0 + 1
        assert np.array_equal(E.pm_get()[0], np.zeros((E.height, E.width), np.float32)), "capture ran the kernel"
        g.replay()
        torch.cuda.synchronize()
        replayed, lab_after = E.pm_get()
        assert np.array_equal(bits(eager), bits(on_stream)) and np.array_equal(bits(eager), bits(replayed))
        assert np.array_equal(bits(lab_after), bits(lab))
    finally:
        E.close()


def test_a_pm_iteration_right_after_the_call():
    """The next launches on the stream see the call's costs: an iteration issued right after it equals the same iteration started
    from lexp_pm_begin(costs, labeling) with the call's costs copied back."""
    from localexpstereo_b200.sweep import PMSweep
    E, _ = _scene_energy()
    S = PMSweep(E, unit_sizes=[5, 15, 25])
    try:
        lab = LC.random_plane_field(E.height, E.width, 0.0, 31.0, 2, beyond=0.05, slope=0.1)
        costs = LC.device_costs(E, lab)
        E.pm_begin(0, labeling=lab)
        E.pm_init_from_labeling(0)
        S.iteration(0, 77)
        a_cost, a_lab = E.pm_get()
        E.pm_begin(0, cost=costs, labeling=lab)
        S.iteration(0, 77)
        b_cost, b_lab = E.pm_get()
        assert np.array_equal(bits(a_cost), bits(b_cost)) and np.array_equal(bits(a_lab), bits(b_lab))
        assert (bits(a_lab) != bits(lab)).any()
    finally:
        S.close()
        E.close()


def test_costs_recomputed_after_post_process():
    """Post-processing changes the labels only: recomputing the costs of the cones crop's post-processed labelings matches the
    oracle, and lexp_energy's data term then equals the oracle's data term of those labelings."""
    import lexp_golden
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import PMSweep
    G = lexp_golden.load()
    prm = L.Parameters(windR=G["windR"], filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.CostVolumeEnergy(G["imL"], G["imR"], G["volL"], G["volR"], prm, G["D"] - 1)
    try:
        E.set_smoothness(1.0, 10.0, 1.0, 0.01)
        for mode in (0, 1):
            S = PMSweep(E, unit_sizes=[6, 18, 40], mode=mode)
            S.begin()
            S.init(seeded_labels(S, 31 + mode))
            S.iteration(0, 500 + mode)
            S.close()
        before = [E.pm_get(m)[1] for m in (0, 1)]
        E.post_process(1.5)
        H, W = E.height, E.width
        ys, xs = LC.all_pixels(H, W)
        for mode in (0, 1):
            lab = E.pm_get(mode)[1]
            assert (bits(lab) != bits(before[mode])).any()
            E.pm_init_from_labeling(mode)
            got, lab2 = E.pm_get(mode)
            assert np.array_equal(bits(lab2), bits(lab))
            ref = LC.c_oracle_costs(G["imR"] if mode else G["imL"], G["volR"] if mode else G["volL"], G["windR"], lab, ys, xs, mode)
            LC.compare(got[ys, xs], ref, f"post-processed view {mode}")
            data, _ = E.energy(mode)
            want = float(ref.astype(np.float64).sum())
            assert abs(data - want) <= 1e-4 * float(np.abs(ref).astype(np.float64).sum()), (data, want)
    finally:
        E.close()


def test_two_rank_cell_shard_copies_are_identical():
    E0, _ = _scene_energy(seed=12)
    E1, _ = _scene_energy(seed=12)
    try:
        lab = LC.random_plane_field(E0.height, E0.width, 0.0, 31.0, 4)
        alone = LC.device_costs(E0, lab)
        for E in (E0, E1):
            E.pm_begin(0, labeling=lab)
        E0.pm_connect_local(0, [E0, E1])
        E1.pm_connect_local(1, [E0, E1])
        E0.pm_init_from_labeling(0)
        E1.pm_init_from_labeling(0)
        c0, l0 = E0.pm_get()
        c1, l1 = E1.pm_get()
        assert np.array_equal(bits(c0), bits(c1)) and np.array_equal(bits(c0), bits(alone))
        assert np.array_equal(bits(l0), bits(lab)) and np.array_equal(bits(l1), bits(lab))
    finally:
        E0.close()
        E1.close()
