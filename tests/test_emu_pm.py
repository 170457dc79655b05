"""tests/test_gpu_pm.py (device-side PatchMatch phase) on the CPU emulator of the kernel source: proposals, fused update,
per-cell completion counters and the host-side schedule, without a GPU (launches run one after the other here, so the
polling of the counters never waits; the ordering itself is exercised on the device by the -m gpu run)."""
import pytest

from emu import emu_lib
import test_gpu_pm as _pm
from lexp_testlib import HostAsDeviceMemory


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
    with emu_lib.emulated():
        yield


@pytest.fixture(scope="module")
def devmem():
    return HostAsDeviceMemory()


def test_emu_pm_phase_replay_small(devmem):
    _pm.test_pm_phase_replay_small(devmem)


def test_emu_pm_phase_replay_r10(devmem):
    _pm.test_pm_phase_replay_r10(devmem)


def test_emu_pm_phase_cell_shard_two_ranks_in_one_process():
    _pm.test_pm_phase_cell_shard_two_ranks_in_one_process()


def test_emu_native_sweep_object_equals_the_python_schedule():
    _pm.test_native_sweep_object_equals_the_python_schedule()


def test_emu_pm_phase_replay_right_view(devmem):
    _pm.test_pm_phase_replay_right_view(devmem)
