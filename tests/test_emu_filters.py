"""The bilateral filter ("BL" / "BF") and the unfiltered mode ("") on the CPU emulator of the kernel source (lexp_filters.cuh): the
unary calls, the warm start and the PatchMatch steps of both energies against the FP64 oracle (tests/filter_checks.py), and a whole
run against the same run issued through the public calls (tests/run_checks.py)."""
import numpy as np
import pytest

import localexpstereo_b200 as L
from emu import emu_lib
import filter_checks as FC
import run_checks as RC
from lexp_testlib import HostAsDeviceMemory

KINDS = [("cv", "bl"), ("cv", "none"), ("naive", "bl"), ("naive", "none")]


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
    with emu_lib.emulated():
        yield


@pytest.fixture(scope="module")
def devmem():
    return HostAsDeviceMemory()


@pytest.mark.parametrize("energy,filt", KINDS)
@pytest.mark.parametrize("mode", [0, 1])
def test_emu_unary_calls(devmem, energy, filt, mode):
    """filterRects at every corner, 1x1 and whole-filterRect targets, steep / NaN / inf planes, every output path."""
    FC.check_unary(devmem, energy, filt, 23, 37, 9, 5, mode=mode, seed=mode)


@pytest.mark.parametrize("windR", [2, 20, 21])
def test_emu_unary_radii(devmem, windR):
    """windR 2 (the smallest), 20 and 21 (windows wider than the staged sub-tile and than the image)."""
    FC.check_unary(devmem, "cv", "bl", 26, 45, 8, windR, seed=windR)


def test_emu_unary_min_disparity(devmem):
    """MIN_DISPARITY != 0: the sampler's slice index is shifted by -MIN."""
    FC.check_unary(devmem, "cv", "none", 17, 30, 12, 4, MIN=2.0, MAX=8.5)
    FC.check_unary(devmem, "cv", "bl", 17, 30, 12, 4, MIN=2.0, MAX=8.5)


@pytest.mark.parametrize("energy,filt", KINDS)
def test_emu_warm_start(energy, filt):
    """Every pixel against the oracle and bit for bit against the unary call (F(p), {p})."""
    FC.check_warm_start(energy, filt, 13, 18, 8, 3, mode=1 if energy == "naive" else 0)


@pytest.mark.parametrize("energy,filt", KINDS)
def test_emu_pm_steps(devmem, energy, filt):
    """An initialisation and a step of every proposer kind on one group: (P), (U), (Q), (I)."""
    FC.check_pm_steps(devmem, energy, filt, 28, 36, 10, 3, unit=4)


@pytest.mark.parametrize("energy,filt", KINDS)
def test_emu_errors(energy, filt):
    FC.check_errors(energy, filt)


def test_emu_filter_names():
    """The names the reference maps to a filter are accepted; those it leaves a null filter for raise."""
    from lexp_testlib import make_scene
    imL, imR, volL, volR = make_scene(8, 10, 4)
    for name in ("GF", "GFfloat", "BL", ""):
        L.CostVolumeEnergy(imL, None, volL, None, L.Parameters(windR=4, filterName=name, filter_param1=10.0), 3).close()
    for name in ("GF", "GFfloat", "BF", ""):
        L.NaiveStereoEnergy(imL, imR, L.Parameters(windR=4, filterName=name, filter_param1=10.0), 3).close()
    for name in ("BF", "bl", "median"):
        with pytest.raises(L.LexpError, match="null pointer"):
            L.CostVolumeEnergy(imL, None, volL, None, L.Parameters(windR=4, filterName=name, filter_param1=10.0), 3)
    for name in ("BL", "gf"):
        with pytest.raises(L.LexpError, match="null pointer"):
            L.NaiveStereoEnergy(imL, imR, L.Parameters(windR=4, filterName=name, filter_param1=10.0), 3)


def _mk(naive, name, H=24, W=32, D=8, windR=3):
    def mk():
        imL, imR, volL, volR = RC.make_scene(H, W, D)
        prm = L.Parameters(windR=windR, filterName=name, filter_param1=10.0, th_col=0.5)
        E = L.NaiveStereoEnergy(imL, imR, prm, D - 1) if naive else L.CostVolumeEnergy(imL, imR, volL, volR, prm, D - 1)
        E.set_smoothness(**RC.SMOOTH)
        return E
    return mk


@pytest.mark.parametrize("naive,name", [(False, "BL"), (False, ""), (True, "BF")])
@pytest.mark.parametrize("views", [(0,), (0, 1)])
def test_emu_run_equals_composition(naive, name, views):
    """lexp_run bit for bit against its public calls; the energy never rises from one graph-cut iteration to the next."""
    lab, raw, calls = RC.check_run_equals_composition(_mk(naive, name), views, 1, 2, [4, 8], RC.PROPS, seed=7)
    for m in views:
        e = [r["energy"] for i, mm, r, _ in calls if mm == m and 1 <= i <= 3]
        assert all(b <= a * (1 + 1e-6) for a, b in zip(e, e[1:])), e
