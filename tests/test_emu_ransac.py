"""tests/test_gpu_ransac.py (the device RansacProposer) on the CPU emulator of the kernel source, bit for bit against
oracle/ransac_oracle.py: the designed units (several batches of samples where the inlier ratio is low), the argument errors, one
small pm iteration (every step certified) and one graph-cut iteration with the reference's proposer lists, and the library's sweep
object against the Python schedule."""
import pytest

from emu import emu_lib
import test_gpu_ransac as _gr
from lexp_testlib import HostAsDeviceMemory, make_scene


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
    with emu_lib.emulated():
        yield


@pytest.fixture(scope="module")
def devmem():
    return HostAsDeviceMemory()


def test_emu_designed_units(devmem):
    _gr.check_designed_units(devmem)


def test_emu_argument_errors():
    _gr.test_argument_errors()


def test_emu_reference_list_iteration(devmem):
    """One pm iteration with the reference's lists, every step certified: every RANSAC proposal bit-identical."""
    H, W, D, windR = 48, 64, 10, 8
    T = _gr.reference_list_pm_iteration(devmem, make_scene(H, W, D), [6, 16, 30], windR)
    assert T.ransac > 30


def test_emu_reference_list_graph_cut_iteration(devmem):
    """One graph-cut iteration with the reference's lists: every RANSAC proposal bit-identical, every RANSAC move certified."""
    H, W, D, windR = 30, 40, 8, 6
    n_r = _gr.reference_list_gc_iteration(devmem, make_scene(H, W, D), [5, 12, 24], D, windR)
    assert n_r > 20


def test_emu_native_sweep_equals_python_with_reference_lists():
    _gr.check_native_equals_python(with_gc=False)   # the graph-cut iteration is slow on the emulator; the GPU test runs it
