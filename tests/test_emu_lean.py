"""The lean build of the fused kernel (three CTAs per SM, windR 20 / 21) on the CPU emulator of the kernel source: against the
two-CTA build bit for bit (check A, also under the reverse and shuffled fiber schedules) and certified against the FP64 oracle
(check B).  See tests/lean_checks.py for the scenes and checks.  Without LEXP_LEAN=1 no emulated launch is large enough to take the
lean build."""
import pytest

from emu import emu_lib
import lean_checks as LC
from lexp_testlib import HostAsDeviceMemory


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
    with emu_lib.emulated():
        yield


@pytest.fixture(scope="module")
def devmem():
    return HostAsDeviceMemory()


DESIGNED = {   # id: (windR, mode, MIN, MAX, LEXP_TILE_OH); about 20 s per check on one CPU core: two scenes per check keep the file
               # near 3 minutes (tests/test_gpu_zz_lean.py runs every combination)
    "r20-left-tall": (20, 0, 0.0, None, 128),
    "r21-right-tall-generic": (21, 1, -4.0, 20.0, 128),
    "r20-right-oh20": (20, 1, 0.0, None, 20),
    "r21-left-oh12-generic": (21, 0, -4.0, 21.0, 12),
}
AB = ["r20-left-tall", "r21-left-oh12-generic"]
CERTIFIED = ["r21-right-tall-generic", "r20-right-oh20"]


def designed(key):
    windR, mode, mn, mx, oh = DESIGNED[key]
    return LC.Designed(windR, mode, mn, mx, oh, seed=len(key))


@pytest.mark.parametrize("key", AB)
def test_emu_lean_equals_two_cta_designed_cells(devmem, monkeypatch, key):
    LC.designed_ab(devmem, monkeypatch, designed(key))


@pytest.mark.parametrize("key", CERTIFIED)
def test_emu_lean_certified_designed_cells(devmem, monkeypatch, key):
    LC.designed_certified(devmem, monkeypatch, designed(key))


@pytest.mark.parametrize("order", [1, 2])
def test_emu_lean_equals_two_cta_fiber_orders(devmem, monkeypatch, order):
    with emu_lib.emulated(order=order):
        LC.designed_ab(devmem, monkeypatch, LC.Designed(20, 0, 0.0, None, 128, seed=order))


SWEEPS = {   # id: (windR, mode, LEXP_TILE_OH)
    "r20-left-oh12": (20, 0, 12),
    "r21-right-oh8": (21, 1, 8),
}


def test_emu_lean_equals_two_cta_sweep(devmem, monkeypatch):
    windR, mode, oh = SWEEPS["r20-left-oh12"]
    LC.sweep_ab(devmem, monkeypatch, LC.SweepScene(windR, mode, tile_oh=oh, seed=3))


def test_emu_lean_certified_sweep(devmem, monkeypatch):
    windR, mode, oh = SWEEPS["r21-right-oh8"]
    LC.sweep_certified(devmem, monkeypatch, LC.SweepScene(windR, mode, tile_oh=oh, seed=3))
