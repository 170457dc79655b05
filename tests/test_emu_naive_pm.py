"""The PatchMatch phase of the image-based energy (tests/naive_pm_checks.py: every step certified against the oracle's update of the
same state) on the CPU emulator of the kernel source, at small sizes: the cones crop at windR 20 with the reference's proposer lists,
the generic-radius instantiation, and planes with v != 0."""
import pytest

from emu import emu_lib
import naive_pm_checks as NP
from lexp_testlib import HostAsDeviceMemory


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
    with emu_lib.emulated():
        yield


@pytest.fixture(scope="module")
def devmem():
    return HostAsDeviceMemory()


@pytest.mark.parametrize("mode", [0, 1])
def test_emu_naive_pm_steps_on_the_cones_crop(devmem, mode):
    NP.scene_cones(devmem, mode, H=56, W=72, units=[5, 15], iterations=1)


def test_emu_naive_pm_steps_at_a_generic_radius(devmem):
    NP.scene_generic_radius(devmem, 0, H=41, W=53, iterations=1)


def test_emu_naive_pm_steps_with_vertical_offsets(devmem):
    NP.scene_vertical_offset(devmem, 1, H=48, W=64)
