"""Large cells of the graph-cut move (layer 2: 3 * 10^5 nodes) run as PHASE KERNELS over all SMs instead of one CTA per cell
(lexp_gc.cuh: lexp_gc_phase_kernel, host loop run_gc_phases).  Same per-node steps, same rounds, same relabelling points: the final
state must be bit-identical to the one-CTA path.  LEXP_GC_BIG_NODES = 0 sends every cell of the test scenes down the phase path.
(Sorted late in the -m gpu suite: the phase path has only run on the emulator so far.)"""
import numpy as np
import pytest

import lexp_replay as G
from lexp_testlib import TorchDeviceMemory

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def devmem():
    return TorchDeviceMemory()


def test_phase_kernels_equal_the_one_cta_path(devmem, monkeypatch):
    import localexpstereo_b200 as L
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 2), (L.PROP_RANDOM, 1)]]
    args = (devmem, 72, 96, 12, 12, [8, 22], props)
    kw = dict(pm_iterations=1, gc_iterations=2, seed=5)
    monkeypatch.delenv("LEXP_GC_BIG_NODES", raising=False)
    one = G.run_gc_replay(*args, **kw)
    monkeypatch.setenv("LEXP_GC_BIG_NODES", "0")       # read by lexp_create
    ph = G.run_gc_replay(*args, **kw)
    assert np.array_equal(one["cost_d"], ph["cost_d"]) and np.array_equal(one["lab_d"], ph["lab_d"])
    G.check_gc_result(ph)    # incl. the minimum-cut energy of every move (block-wise double sums instead of thread-wise ones)


def test_phase_kernels_mixed_sizes_and_strong_smoothness(devmem, monkeypatch):
    """Threshold between the layers' cell sizes: layer 0 (24 x 24 nodes) on the one-CTA kernel, layer 1 (66 x 66) as phases; large lambda."""
    import localexpstereo_b200 as L
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)], [(L.PROP_EXPANSION, 1)]]
    smooth = dict(lam=5.0, omega=4.0, th_smooth=1.5, epsilon=0.05)
    args = (devmem, 60, 80, 10, 12, [8, 22], props)
    kw = dict(pm_iterations=0, gc_iterations=1, seed=11, mode=1, smooth=smooth)
    monkeypatch.delenv("LEXP_GC_BIG_NODES", raising=False)
    one = G.run_gc_replay(*args, **kw)
    monkeypatch.setenv("LEXP_GC_BIG_NODES", "1000")
    ph = G.run_gc_replay(*args, **kw)
    assert np.array_equal(one["cost_d"], ph["cost_d"]) and np.array_equal(one["lab_d"], ph["lab_d"])
    G.check_gc_result(ph)
