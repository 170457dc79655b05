"""Every PatchMatch step of the cost-volume energy on the device against the oracle's update of the SAME state: tests/pm_step_rig.py
certifies each step without a budget -- (P) the proposal, (U) the update rule bit for bit, (Q) the proposal cost against the FP64 C
oracle on every target pixel, (I) the PatchMatch cost equals the unary instantiation's -- and the states carry pixel tags, so every
proposal names the pixel it was drawn from.  Designed scenes (ragged units, the update rule at its edges, MIN / MAX that take the
generic sampler, many work items per cell, RandomProposer at the ends of m), the benchmark's workload layer by layer and two sizes.
(Sorted after the graph-cut tests and before the large-size tests.)"""
import time

import numpy as np
import pytest

from oracle import lexp_oracle as O
from lexp_testlib import TorchDeviceMemory, bits, make_scene, seeded_labels
from pm_step_rig import Rig, Tally, assert_same_state, run_sweep

pytestmark = pytest.mark.gpu

INVALID = np.float32(O.COST_FOR_INVALID)


@pytest.fixture(scope="module")
def devmem():
    return TorchDeviceMemory()


# ---- designed scenes (small) -------------------------------------------------------------------------------------------------------------
def small_rig(devmem, H, W, D, windR, units, proposers, mode=0, seed=0, MIN=0.0, MAX=None):
    imL, imR, volL, volR = make_scene(H, W, D, seed=seed)
    return Rig(devmem, imL, imR, volL, volR, windR, units, proposers, mode, MIN, MAX)


def scene_tags(devmem, mode=0):
    """A ragged image (the last unit of every row and column is narrower), two layers, Expansion and Random, two iterations, the
    state tagged after the initialisation: every proposal names its source pixel."""
    import localexpstereo_b200 as L
    H, W, D = 67, 89, 12
    R = small_rig(devmem, H, W, D, 12, [7, 19], [[(L.PROP_EXPANSION, 2), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]],
                  mode, seed=3)
    try:
        for lay in R.S.lm.layers:
            us = lay.unitRegions
            assert min(u[2] for u in us) < lay.regionUnitSize and min(u[3] for u in us) < lay.regionUnitSize, "the image should be ragged"
        T = run_sweep(R, seeded_labels(R.S, 21), 2, 5, what=f"pixel tags, mode {mode}")
        assert T.n_exact > 300 and T.n_random > 300 and T.named > 0
        return T
    finally:
        R.close()


def scene_update_edges(devmem, mode=0):
    """PROP_LIST steps on designed states: ties, the next float above q, NaN, +inf and COST_FOR_INVALID against an invalid plane, a
    NaN plane."""
    import localexpstereo_b200 as L
    H, W, D = 40, 56, 12
    R = small_rig(devmem, H, W, D, 12, [8], [[(L.PROP_EXPANSION, 1)]], mode, seed=8)
    try:
        S = R.S
        R.Eq.pm_begin(mode)
        (_, _, g, _), (_, _, gq, _) = S.schedule[5], R.Sq.schedule[5]
        n = g.plan.num_calls
        old = np.zeros((H, W, 4), np.float32)
        old[..., 2] = 3.0
        rs = np.random.default_rng(mode)
        good = np.stack([[rs.uniform(-0.05, 0.05), rs.uniform(-0.05, 0.05), rs.uniform(4, 7), 7.0] for _ in range(n)]).astype(np.float32)
        far = np.tile(np.float32([0, 0, -50, 1]), (n, 1))
        nanp = np.tile(np.float32([np.nan, 0, 5, 2]), (n, 1))

        def step(cost, planes):
            R.E.pm_reset_sync()
            R.E.pm_begin(mode, cost, old)
            pre, post, inside, q = R.certify(g, gq.plan, L.PROP_LIST, planes=planes)
            changed = (bits(post[0]) != bits(pre[0])) | (bits(post[1]) != bits(pre[1])).any(axis=2)
            return inside, q, changed

        inf = np.full((H, W), np.inf, np.float32)
        inside, q, changed = step(inf, good)                  # +inf: every target pixel takes the plane
        assert np.array_equal(changed, inside) and (q != INVALID).all()
        qimg = np.ones((H, W), np.float32)
        qimg[inside] = q
        assert not step(qimg, good)[2].any(), "a tie (cur == q) must not update"
        _, _, changed = step(np.nextafter(qimg, np.float32(np.inf)), good)
        assert np.array_equal(changed, inside), "cur = nextafter(q, +inf) must update every target pixel"
        assert not step(np.full((H, W), np.nan, np.float32), good)[2].any(), "a NaN current cost must never update"
        _, q, changed = step(inf, far)
        assert (q == INVALID).all() and np.array_equal(changed, inside), "+inf against COST_FOR_INVALID must update"
        assert not step(np.full((H, W), INVALID, np.float32), far)[2].any(), "COST_FOR_INVALID against COST_FOR_INVALID must not update"
        mixed = np.where(rs.random((H, W)) < 0.5, np.float32(np.inf), np.float32(0.5))
        step(mixed, nanp)                                      # a NaN plane: whatever q the oracle gives it, the rule holds
        print(R.T.line(f"update edges, mode {mode}"))
    finally:
        R.close()


def scene_min_max(devmem, mn, mx):
    """MIN_DISPARITY != 0 or MAX_DISPARITY != D - 1: the generic sampler inside the PatchMatch kernel and RandomProposer's clamps."""
    import localexpstereo_b200 as L
    H, W, D = 48, 70, 16
    R = small_rig(devmem, H, W, D, 12, [8, 20], [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 3)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)]],
                  seed=77, MIN=mn, MAX=mx)
    try:
        run_sweep(R, seeded_labels(R.S, 13), 1, 9, what=f"MIN {mn}, MAX {mx}")
    finally:
        R.close()


def scene_many_items(devmem):
    """Every layer-1 cell cut into >= 32 work items (LEXP_TILE_OH = 8, set by the caller before the contexts exist): the proposal
    hand-over through the cell's ticket, ready flag and plane."""
    import localexpstereo_b200 as L
    H, W, D = 140, 150, 12
    R = small_rig(devmem, H, W, D, 12, [19, 64], [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]],
                  seed=4)
    try:
        items = [g.plan.num_items / g.plan.num_calls for g in R.S.groups if g.layer == 1]
        assert min(items) >= 32, items
        run_sweep(R, seeded_labels(R.S, 17), 1, 3, what=f"{min(items):.0f} work items per layer-1 cell")
    finally:
        R.close()


def scene_random_m(devmem, mode=1):
    """Direct RandomProposer steps with m = 0, 1 and 120 (the C-ABI's bound: exp2f(-121) is still a normal float) on a tagged state,
    with the random streams of the sweep's three RandomProposer steps of iteration 0 (seed 8)."""
    import localexpstereo_b200 as L
    H, W, D = 44, 60, 12
    R = small_rig(devmem, H, W, D, 12, [8], [[(L.PROP_RANDOM, 3)]], mode, seed=6)
    try:
        S = R.S
        R.Eq.pm_begin(mode)
        R.E.pm_begin(mode)
        R.init(seeded_labels(S, 31))
        R.tag(R.E)
        for (li, gi, g, _), (_, _, gq, _) in list(zip(S.schedule, R.Sq.schedule))[:8]:
            R.E.pm_reset_sync()
            for (k, kind, _, sd), m in zip(S.group_steps(li, gi, 0, 8), (0, 1, 120)):
                R.certify(g, gq.plan, kind, m, sd, k)
        print(R.T.line(f"Random at m = 0, 1, 120, mode {mode}"))
        assert R.T.n_random > 80 and R.T.named > 0
    finally:
        R.close()


# ---- tests: designed scenes --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [0, 1])
def test_pixel_tags_name_every_source_pixel(devmem, mode):
    scene_tags(devmem, mode)


@pytest.mark.parametrize("mode", [0, 1])
def test_update_rule_at_its_edges(devmem, mode):
    scene_update_edges(devmem, mode)


@pytest.mark.parametrize("mn,mx", [(-4.0, 11.0), (0.0, 9.0)])
def test_nonzero_min_and_short_max_disparity(devmem, mn, mx):
    scene_min_max(devmem, mn, mx)


def test_many_work_items_per_cell(devmem, monkeypatch):
    monkeypatch.setenv("LEXP_TILE_OH", "8")
    scene_many_items(devmem)


def test_random_proposer_at_the_ends_of_m(devmem):
    scene_random_m(devmem, mode=1)


# ---- at scale -----------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bench_rig(devmem):
    """bench.py's PatchMatch-phase workload: 2048 x 1536 x 256, windR 20, V3_PROPOSERS_DEVICE, initial labels of bench.py (seed 99),
    the volume drawn on the device (torch.rand, seed 1234) and copied to the host for the C oracle (3.2 GB)."""
    import torch
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import V3_PROPOSERS_DEVICE
    W, H, D, windR = 2048, 1536, 256, 20
    imL = synth.synthetic_image(H, W, 42)
    vol = torch.rand((D, H, W), generator=torch.Generator(device="cuda").manual_seed(1234), device="cuda", dtype=torch.float32)
    torch.cuda.synchronize()
    R = Rig(devmem, imL, None, vol, None, windR, None, V3_PROPOSERS_DEVICE, vol_host=vol.cpu().numpy())
    del vol
    torch.cuda.empty_cache()
    units = R.S.lm.layers[0].unitRegions
    labels = synth.synthetic_planes([units[i] for i in range(len(units))], 1, D, 99)[0][R.S.init_index]
    yield R, labels
    R.close()


BENCH_SEED = 4321
BENCH_REPLAYED = 3   # bench.py's default --warmup: the iteration index it captures and replays


@pytest.mark.parametrize("it,layer", [(None, None)] + [(it, li) for it in (0, BENCH_REPLAYED) for li in range(3)])
def test_every_step_of_the_benchmark_workload(bench_rig, it, layer):
    """The initialisation (it = None), or every step of one layer of iteration `it` after iterations 0 .. it - 1 and the layer's
    predecessors ran uninterrupted; the state tagged after the initialisation on both contexts.  The state at the end of the layer
    must equal the twin's uninterrupted sweep."""
    R, labels = bench_rig
    R.T, R.tagged, R.tag_check_pending = Tally(), False, False
    t0 = time.perf_counter()
    ref = R.twin_reference(labels, BENCH_SEED, None if it is None else (it, layer), tag=True)
    R.E.pm_begin(0)
    R.init(labels, certify=it is None)
    R.tag(R.E)
    if it is None:
        state = R.get(R.E)
    else:
        for i in range(it):
            R.iteration(i, BENCH_SEED, certify=lambda g: False)
        state = R.iteration(it, BENCH_SEED, certify=lambda g: g.layer == layer, snap_layer=layer)[1]
    what = "benchmark workload, " + ("initialisation" if it is None else f"iteration {it}, layer {layer}")
    assert_same_state(state, ref, what)
    print(R.T.line(what) + f"; {time.perf_counter() - t0:.1f} s in all")
    assert R.T.steps == (1 if it is None else 16 * (9 if layer == 0 else 3))


def scene_at_size(devmem, W, H, D, windR, mode, seed):
    """Two iterations of V3_PROPOSERS_DEVICE on a synthetic scene, every step certified, the state tagged after the initialisation."""
    from localexpstereo_b200.sweep import V3_PROPOSERS_DEVICE
    imL, imR, volL, volR = make_scene(H, W, D, seed=seed)
    R = Rig(devmem, imL, imR if mode else None, volL, volR if mode else None, windR, None, V3_PROPOSERS_DEVICE, mode)
    try:
        t0 = time.perf_counter()
        run_sweep(R, seeded_labels(R.S, seed), 2, 1000 + seed, what=f"{W} x {H} x {D}, windR {windR}, mode {mode}")
        print(f"  {time.perf_counter() - t0:.1f} s in all")
    finally:
        R.close()


def test_every_step_of_the_r16_instantiation(devmem):
    scene_at_size(devmem, 960, 544, 96, 32, 0, 5)


def test_every_step_of_the_generic_radius_right_view(devmem):
    scene_at_size(devmem, 437, 291, 40, 12, 1, 6)
