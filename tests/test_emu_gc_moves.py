"""tests/test_gpu_zz_gc_moves.py (every graph-cut move against the exact minimum cut of the same graph) on the CPU emulator of the
kernel source: the lambda = 0, free-node, geometry and COST_FOR_INVALID-dominated scenes, a 40 x 40 corridor, and the phase kernels
against the one-CTA kernel on a small scene."""
import os

import pytest

from emu import emu_lib
import test_gpu_zz_gc_moves as _mv
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


@pytest.mark.parametrize("mode", [0, 1])
def test_emu_lambda_zero_is_the_closed_form(devmem, mode):
    _mv.test_lambda_zero_is_the_closed_form(devmem, mode)


@pytest.mark.parametrize("mode", [0, 1])
def test_emu_free_nodes_take_the_proposal(devmem, mode):
    _mv.test_free_nodes_take_the_proposal(devmem, mode)


def test_emu_invalid_dominated_cells(devmem):
    _mv.test_invalid_dominated_cells(devmem)


@pytest.mark.parametrize("mode", [0, 1])
def test_emu_cells_at_corners_edges_and_the_whole_image(devmem, mode):
    _mv.test_cells_at_corners_edges_and_the_whole_image(devmem, mode)


def test_emu_long_residual_path(devmem, monkeypatch):
    monkeypatch.delenv("LEXP_GC_BIG_NODES", raising=False)
    r = _mv.scene_corridor(devmem, 40, 40)
    assert r["path"] > 100


def test_emu_phase_kernels_equal_the_one_cta_kernel(devmem, monkeypatch):
    _mv.schedule_variants(devmem, monkeypatch, "geometry", [(None, "0")])
