"""tests/test_gpu_zz_pm_steps.py (every PatchMatch step against the oracle's update of the same state) on the CPU emulator of the
kernel source: pixel tags, the update rule at its edges, MIN / MAX disparities that take the generic sampler, many work items per
cell and RandomProposer at the ends of m."""
import pytest

from emu import emu_lib
import test_gpu_zz_pm_steps as _ps
from lexp_testlib import HostAsDeviceMemory


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
    with emu_lib.emulated():
        yield


@pytest.fixture(scope="module")
def devmem():
    return HostAsDeviceMemory()


@pytest.mark.parametrize("mode", [0, 1])
def test_emu_pixel_tags_name_every_source_pixel(devmem, mode):
    _ps.scene_tags(devmem, mode)


@pytest.mark.parametrize("mode", [0, 1])
def test_emu_update_rule_at_its_edges(devmem, mode):
    _ps.scene_update_edges(devmem, mode)


@pytest.mark.parametrize("mn,mx", [(-4.0, 11.0), (0.0, 9.0)])
def test_emu_nonzero_min_and_short_max_disparity(devmem, mn, mx):
    _ps.scene_min_max(devmem, mn, mx)


def test_emu_many_work_items_per_cell(devmem, monkeypatch):
    monkeypatch.setenv("LEXP_TILE_OH", "8")
    _ps.scene_many_items(devmem)


def test_emu_random_proposer_at_the_ends_of_m(devmem):
    _ps.scene_random_m(devmem, mode=1)
