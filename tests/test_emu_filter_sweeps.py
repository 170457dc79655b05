"""Whole PatchMatch sweeps with the bilateral filter ("BL" / "BF") and the unfiltered mode ("") on the CPU emulator of the kernel
source, every step certified by tests/pm_step_rig.py and the final state equal to the twin's uninterrupted sweep bit for bit
(tests/test_gpu_zz_filter_scale.py's scenes at small sizes): both energies, both views, the reference's proposer lists (RANSAC
included) -- so the decomposed step (proposals, the unary costs into the view's proposal-cost image, the update kernel) is held to
the right view's guide, volume and state across groups whose filterRects overlap -- and cells cut into several work items."""
import pytest

from emu import emu_lib
import test_gpu_zz_filter_scale as _fs
from lexp_testlib import HostAsDeviceMemory


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
    with emu_lib.emulated():
        yield


@pytest.fixture(scope="module")
def devmem():
    return HostAsDeviceMemory()


def _reference_lists(n):
    from localexpstereo_b200.sweep import V3_PROPOSERS_REFERENCE
    return V3_PROPOSERS_REFERENCE[:n]


@pytest.mark.parametrize("energy,filt", [("cv", "BL"), ("cv", ""), ("naive", "BF")])
@pytest.mark.parametrize("mode", [0, 1])
def test_emu_filter_sweep(devmem, energy, filt, mode):
    T = _fs.scene_filter_sweep(devmem, energy, filt, mode, 37, 53, 10, 4, [4, 12], _reference_lists(2), iterations=1, seed=mode)
    assert T.ransac > 0 and T.n_random > 0 and T.q_cells >= T.steps


def test_emu_filter_sweep_many_work_items_per_cell(devmem, monkeypatch):
    """LEXP_TILE_OH = 8 (before the contexts exist): every layer-1 cell spans several work items of the unary kernel, whose items
    read their own tile origin and compact-output offset."""
    monkeypatch.setenv("LEXP_TILE_OH", "8")
    import localexpstereo_b200 as L
    from lexp_testlib import make_scene
    from pm_step_rig import Rig, run_sweep
    from lexp_testlib import seeded_labels
    imL, imR, volL, volR = make_scene(60, 70, 10, seed=4)
    R = Rig(devmem, imL, imR, volL, volR, 4, [6, 24], _reference_lists(2), 1, filter="BL", sig2=_fs.SIG2)
    try:
        items = [g.plan.num_items / g.plan.num_calls for g in R.S.groups if g.layer == 1]
        assert min(items) >= 4, items
        T = run_sweep(R, seeded_labels(R.S, 17), 1, 3, what=f"'BL' mode 1, {min(items):.0f} work items per layer-1 cell")
        assert T.ransac > 0
    finally:
        R.close()
