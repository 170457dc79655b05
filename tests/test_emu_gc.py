"""tests/test_gpu_zz_gc.py (pairwise terms + graph-cut move on the device) on the CPU emulator of the kernel source: the graph
construction, the deterministic push-relabel and the host-side schedule, without a GPU."""
import pytest

from emu import emu_lib
import test_gpu_zz_gc as _gc
import test_gpu_zz_gc_phases as _ph
from lexp_replay import SMOOTH, check_gc_result, recording, run_gc_replay
from lexp_testlib import HostAsDeviceMemory, make_scene


@pytest.fixture(scope="module", autouse=True)
def _use_emulator(monkeypatch_module=None):
    import os
    prev = os.environ.get("LEXP_GC_THREADS")
    os.environ["LEXP_GC_THREADS"] = "128"   # fibers per emulated CTA: fewer context switches per barrier, same arithmetic
    with emu_lib.emulated():
        yield
    if prev is None:
        os.environ.pop("LEXP_GC_THREADS", None)
    else:
        os.environ["LEXP_GC_THREADS"] = prev


@pytest.fixture(scope="module")
def devmem():
    return HostAsDeviceMemory()


def test_emu_smoothness_coefficients():
    _gc.test_smoothness_coefficients_equal_the_oracle()


def test_emu_pairwise_terms():
    _gc.test_pairwise_terms_equal_the_oracle_bit_for_bit()


def test_emu_gc_replay_small(devmem):
    import localexpstereo_b200 as L   # the GPU test's scene with one graph-cut iteration instead of two (emulation time)
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 2), (L.PROP_RANDOM, 1)]]
    check_gc_result(run_gc_replay(devmem, 72, 96, 12, 12, [8, 22], props, pm_iterations=1, gc_iterations=1, seed=5))


def test_emu_gc_replay_right_view_strong_smoothness(devmem):
    _gc.test_gc_replay_right_view_strong_smoothness(devmem)


def test_emu_gc_moves_never_raise_the_energy(devmem):
    _gc.test_gc_moves_never_raise_the_energy(devmem)


# (_ph.test_phase_kernels_equal_the_one_cta_path -- every cell on the phase path, two iterations -- takes four minutes of fiber
#  switches here; it was run on the emulator when the path was written and is part of the -m gpu suite)
def test_emu_phase_kernels_mixed_sizes(devmem, monkeypatch):
    _ph.test_phase_kernels_mixed_sizes_and_strong_smoothness(devmem, monkeypatch)


def test_emu_gc_result_does_not_depend_on_the_thread_schedule(devmem):
    """The graph-cut move is deterministic by construction (push slots instead of atomics, relabels computed from the heights of the
    round's start): forward, reverse and reshuffled-every-pass schedules of the emulated threads must give the same state and the same
    minimum-cut energies bit for bit -- a missing barrier or an order-dependent read in lexp_gc_move_kernel would show here."""
    import numpy as np
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import GCSweep
    from oracle import lexp_oracle as O
    H, W, D, windR = 48, 64, 10, 12
    imL, _, volL, _ = make_scene(H, W, D, seed=4)
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]]
    outs = []
    for order in (0, 1, 2):
        with emu_lib.emulated(order=order):
            E = L.CostVolumeEnergy(imL, None, volL, None, L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5), D - 1)
            S = GCSweep(E, unit_sizes=[8], proposers=props, **SMOOTH)
            rng = O.CvRNG(3)
            S.begin()
            S.init(np.stack([O.create_random_label(rng, u[0], u[1], 0.0, D - 1.0) for u in S.init_units]))
            flows = recording(devmem, S, 0, 21, gc=True)[1]
            S.gc_iteration(0, 21, flows_out={k: devmem.ptr(v) for k, v in flows.items()})
            cost, lab = S.get()
            outs.append((cost, lab, np.concatenate([np.ascontiguousarray(v).view(np.float64).ravel() for v in flows.values()])))
            S.close(); E.close()
    for o in outs[1:]:
        assert np.array_equal(outs[0][0], o[0]) and np.array_equal(outs[0][1], o[1]) and np.array_equal(outs[0][2], o[2])
    assert (outs[0][2] != 0).any()


def test_emu_gc_iteration_on_the_image_based_energy(devmem):
    _gc.test_gc_iteration_on_the_image_based_energy(devmem)


@pytest.mark.parametrize("naive", [False, True])
def test_emu_native_sweep_object_runs_the_same_graph_cut_iteration(naive):
    _gc.test_native_sweep_object_runs_the_same_graph_cut_iteration(naive)
