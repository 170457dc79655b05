"""tests/test_gpu_zz_gc_scale.py on the CPU emulator of the kernel source: the round limit (LEXP_GC_MAX_ROUNDS) in both execution forms
on a 40 x 40 corridor, one plan of 49 cells on the phase kernels, the subnormal coefficient scene, and the certified graph-cut iteration of the image-based energy at a small size."""
import os

import pytest

from emu import emu_lib
import test_gpu_zz_gc_scale as _sc
from lexp_testlib import HostAsDeviceMemory


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
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


def test_emu_round_limit(devmem, monkeypatch):
    _sc.round_limit_forms(devmem, monkeypatch, (0, 24), 40, 40)


@pytest.mark.parametrize("mode", [0, 1])
def test_emu_subnormal_coefficients_and_moves(devmem, monkeypatch, mode):
    _sc.test_subnormal_coefficients_and_moves(devmem, monkeypatch, mode)


def test_emu_many_cells_on_the_phase_kernels(devmem):
    _sc.test_many_cells_on_the_phase_kernels(devmem)


def test_emu_image_based_energy(devmem, monkeypatch):
    monkeypatch.delenv("LEXP_GC_BIG_NODES", raising=False)
    T = _sc.scene_image_based(devmem, 96, 72, 16, (5, 15, 25), pm_iterations=1)
    assert T.moves > 100
