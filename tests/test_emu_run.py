"""A whole run (lexp_run, the random-start kernel and the device evaluator) on the CPU emulator of the kernel source.  The emulator
evaluates sin / cos with the host's libm, so the random start equals the oracle bit for bit here."""
import numpy as np
import pytest

from emu import emu_lib
import run_checks as RC


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
    import os
    prev = os.environ.get("LEXP_GC_THREADS")
    os.environ["LEXP_GC_THREADS"] = "128"
    with emu_lib.emulated():
        yield
    if prev is None:
        os.environ.pop("LEXP_GC_THREADS", None)
    else:
        os.environ["LEXP_GC_THREADS"] = prev


@pytest.mark.parametrize("naive", [False, True])
def test_emu_random_start_equals_the_oracle(naive):
    E = RC.scene_energy(40, 56, 10, 6, naive=naive)
    try:
        RC.check_random_start(E, [8, 16], seed=77)
        RC.check_random_start(E, [5], seed=2**63 + 5)
    finally:
        E.close()


def test_emu_evaluator_counts_equal_numpy():
    E = RC.scene_energy(40, 56, 10, 6)
    try:
        gt, nonocc = RC.synthetic_gt(E, 3)
        RC.check_random_start(E, [8], seed=4)
        RC.check_evaluate(E, gt, nonocc)
        gt[:] = np.inf                         # no valid pixel, every pixel masked out: the rates are NaN as in the reference
        RC.check_evaluate(E, gt, np.zeros_like(nonocc))
    finally:
        E.close()


@pytest.mark.parametrize("naive,views,given", [(False, (0,), False), (False, (0, 1), False), (False, (0, 1), True), (True, (0, 1), False)])
def test_emu_run_equals_the_composed_run(naive, views, given):
    mk = lambda: RC.scene_energy(32, 48, 10, 6, naive=naive)
    RC.check_run_equals_composition(mk, views, 1, 1, [8, 16], RC.PROPS, seed=11, given=given)


def test_emu_run_seeds_are_distinct_and_match_the_library():
    from localexpstereo_b200 import _capi
    from localexpstereo_b200.sweep import RUN_GC, RUN_INIT, RUN_PM, run_seed
    seeds = set()
    for base in (0, 1, 12345, 2**64 - 1):
        for m in (0, 1):
            keys = [(RUN_INIT, 0)] + [(p, it) for p in (RUN_PM, RUN_GC) for it in range(8)]
            for p, it in keys:
                s = run_seed(base, m, p, it)
                assert s == _capi.lib().lexp_run_seed(base, m, p, it)
                seeds.add(s)
            assert run_seed(base, m, RUN_INIT, 0) == run_seed(base, m, RUN_INIT, 5)
    assert len(seeds) == 4 * 2 * 17
