"""The launch-chain tests of tests/test_gpu_launch_chains.py that need no CUDA graph and no torch stream, on the emulator.

The emulator runs launches one after another and compiles programmatic dependent launch out, so the comparison with the PDL-off
context is trivial here and no launch is counted as overlapped.  What runs is the rest of each test: the per-launch composition in
issue order, the check that consecutive writes are distinguishable, the oracle on the pixels each group's last step leaves behind,
and the interleaving of host-plane calls with a device-plane sweep -- on scenes small enough for the emulator, with the same
kinds of edges (a ragged generic-R cost-volume case and the image-based energy)."""
import pytest

from emu import emu_lib

import test_gpu_launch_chains as _c
from lexp_testlib import HostAsDeviceMemory

# W not a multiple of 4, generic R; three layers and K = 3 / 2 / 2 steps keep the launch count small
SCENES = {
    "ragged_61x45x32_r12": dict(W=61, H=45, D=32, windR=12, units=[6, 13, 22], steps=[3, 2, 2]),
    "naive_64x48x16_r20": dict(W=64, H=48, D=16, windR=20, naive=True, units=[5, 15, 25], steps=[3, 2, 2]),
}


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
    with emu_lib.emulated():
        yield


@pytest.fixture(scope="module")
def devmem():
    return HostAsDeviceMemory()


@pytest.fixture(scope="module")
def expect_overlap():
    return False


@pytest.fixture(scope="module")
def scene_cache(devmem, _use_emulator):
    cache = {}
    yield lambda name: cache.get(name) or cache.setdefault(name, _c.Scene(devmem, None, **SCENES[name]))
    for sc in cache.values():
        sc.close()


@pytest.fixture(params=list(SCENES))
def scene(request, scene_cache):
    return scene_cache(request.param)


small_scene = scene

test_emu_unary_sweep_overlapped_equals_serialized = _c.test_unary_sweep_overlapped_on_a_caller_stream_equals_serialized
test_emu_unary_sweep_last_writer_wins = _c.test_unary_sweep_last_writer_wins
test_emu_host_planes_between_overlapped_launches = _c.test_host_planes_between_overlapped_launches
