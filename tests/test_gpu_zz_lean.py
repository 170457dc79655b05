"""The lean build of the fused kernel (lexp_fused_kernel<10, false, true, kLeanCtas>: three CTAs per SM, at most 56 registers) on
the H100, where its register budget and load scoreboard run for real: against the two-CTA build bit for bit (check A) and certified
against the FP64 oracle (check B) on the designed cells and sweeps of tests/lean_checks.py, and the benchmark's workload at scale
with LEXP_LEAN=1, =0 and unset.
At scale the lean launches per layer with LEXP_LEAN unset are those the rule gives the planner's items: the initialisation, all 144
launches of layer 0 and all 48 of layer 1, and 6 of the 48 launches of layer 2 (2 of its 16 groups).
(Sorted after the graph-cut tests and before the large-size tests.  About 20 s on an H100 80GB HBM3, 5 s of it the workload at scale.)"""
import time

import numpy as np
import pytest

import lean_checks as LC
from lexp_testlib import TorchDeviceMemory

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def devmem():
    return TorchDeviceMemory()


DESIGNED = {   # id: (windR, mode, MIN, MAX, LEXP_TILE_OH)
    "r20-left-tall": (20, 0, 0.0, None, 128),
    "r20-right-tall": (20, 1, 0.0, None, 128),
    "r21-left-tall": (21, 0, 0.0, None, 128),
    "r21-right-tall-generic": (21, 1, -4.0, 20.0, 128),
    "r20-left-oh8": (20, 0, 0.0, None, 8),
    "r20-right-oh20": (20, 1, 0.0, None, 20),
    "r21-left-oh12-generic": (21, 0, -4.0, 21.0, 12),
    "r21-right-oh8-generic": (21, 1, -4.0, 22.0, 8),
}


def designed(key):
    windR, mode, mn, mx, oh = DESIGNED[key]
    return LC.Designed(windR, mode, mn, mx, oh, seed=len(key))


@pytest.mark.parametrize("key", list(DESIGNED))
def test_lean_equals_two_cta_designed_cells(devmem, monkeypatch, key):
    LC.designed_ab(devmem, monkeypatch, designed(key))


@pytest.mark.parametrize("key", list(DESIGNED))
def test_lean_certified_designed_cells(devmem, monkeypatch, key):
    LC.designed_certified(devmem, monkeypatch, designed(key))


SWEEPS = {   # id: (windR, mode, LEXP_TILE_OH, MIN, MAX)
    "r20-left-oh12": (20, 0, 12, 0.0, None),
    "r21-right-oh8": (21, 1, 8, 0.0, None),
    "r20-right-oh20-generic": (20, 1, 20, -4.0, 13.0),
    "r21-left-oh128": (21, 0, 128, 0.0, None),
}


def sweep(key):
    windR, mode, oh, mn, mx = SWEEPS[key]
    if oh == 128:   # targets of at least 128 rows: full-height tiles, cones of 168 rows
        return LC.SweepScene(windR, mode, mn, mx, tile_oh=oh, seed=4, H=330, W=250, D=20, units=(44, 96))
    return LC.SweepScene(windR, mode, mn, mx, tile_oh=oh, seed=3)


@pytest.mark.parametrize("key", list(SWEEPS))
def test_lean_equals_two_cta_sweep(devmem, monkeypatch, key):
    LC.sweep_ab(devmem, monkeypatch, sweep(key), iterations=2)


@pytest.mark.parametrize("key", list(SWEEPS))
def test_lean_certified_sweep(devmem, monkeypatch, key):
    LC.sweep_certified(devmem, monkeypatch, sweep(key), iterations=2)


# ---- at scale ---------------------------------------------------------------------------------------------------------------------------
BENCH_SEED = 4321


@pytest.fixture(scope="module")
def bench_trio(devmem):
    """bench.py's PatchMatch-phase workload (2048 x 1536 x 256, windR 20, V3_PROPOSERS_DEVICE, the initial labels of bench.py, the
    volume drawn on the device with seed 1234) on three contexts: LEXP_LEAN=1, =0 and unset (3.2 GB of volume each)."""
    import torch
    import localexpstereo_b200 as L
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import PMSweep, V3_PROPOSERS_DEVICE
    W, H, D, windR = 2048, 1536, 256, 20
    imL = synth.synthetic_image(H, W, 42)
    vol = torch.rand((D, H, W), generator=torch.Generator(device="cuda").manual_seed(1234), device="cuda", dtype=torch.float32)
    torch.cuda.synchronize()
    mp = pytest.MonkeyPatch()
    sweeps = {}
    try:
        for lean in (1, 0, None):
            E = LC.under_lean(mp, lean, lambda: L.CostVolumeEnergy(imL, None, vol, None, LC.params(windR), D - 1))
            sweeps[lean] = PMSweep(E, proposers=V3_PROPOSERS_DEVICE)
        del vol
        torch.cuda.empty_cache()
        S = sweeps[1]
        units = S.lm.layers[0].unitRegions
        labels = synth.synthetic_planes([units[i] for i in range(len(units))], 1, D, 99)[0][S.init_index]
        yield sweeps, labels
    finally:
        mp.undo()
        for S in sweeps.values():
            S.close()
            S.energy.close()


def test_benchmark_workload_lean_equals_two_cta(devmem, bench_trio):
    """The initialisation and iteration 0, one group at a time on all three contexts: bit-identical states and recorded planes after
    every group.  LEXP_LEAN=1 adds the launches the shipped rule keeps on the two-CTA build (most of layer 2: tall items up to 64 wide,
    several per cell).  With LEXP_LEAN unset, the lean launches per layer must be those of the rule (LC.shipped_rule_is_lean on the
    planner's items)."""
    import torch
    sweeps, labels = bench_trio
    num_sms = torch.cuda.get_device_properties(0).multi_processor_count
    Su, E1, E0, Eu = sweeps[None], sweeps[1].energy, sweeps[0].energy, sweeps[None].energy
    expect, plan_lean = {}, {}
    for grp in ([Su.init_group] + Su.groups):
        items = LC.plan_items(grp.filters, grp.targets, LC.R10, None, num_sms)
        assert grp.plan.num_items == len(items), "the planner replica disagrees"
        plan_lean[id(grp.plan)] = LC.shipped_rule_is_lean(items, num_sms)
    expect[(None, 0)] = int(plan_lean[id(Su.init_plan)])
    for (li, gi, g, _) in Su.schedule:
        expect[(0, li)] = expect.get((0, li), 0) + plan_lean[id(g.plan)] * len(Su.group_steps(li, gi, 0, BENCH_SEED))
    seen, last = {}, [Eu.lean_launch_count]

    def layer_end(it, li):
        seen[(it, li)] = Eu.lean_launch_count - last[0]
        last[0] = Eu.lean_launch_count

    t0 = time.perf_counter()
    launches = LC.compare_walks(devmem, sweeps, labels, 1, BENCH_SEED, on_layer_end=layer_end)
    t = time.perf_counter() - t0
    for key in sorted(launches, key=lambda k: (-1, 0) if k[0] is None else k):
        print(f"{'initialisation' if key[0] is None else f'iteration {key[0]}, layer {key[1]}'}: {launches[key]} launches, "
              f"{seen[key]} lean with LEXP_LEAN unset (rule: {expect[key]})")
    print(f"  {t:.1f} s")
    assert E1.lean_launch_count == sum(launches.values()) and E0.lean_launch_count == 0
    assert seen == expect
    # layers 0 and 1 of this workload run lean throughout, layer 2 mostly on the two-CTA build
    assert seen[(0, 0)] == launches[(0, 0)] and seen[(0, 1)] == launches[(0, 1)] and 0 < seen[(0, 2)] < launches[(0, 2)]
