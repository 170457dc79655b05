"""lexp_pm_init_from_labeling (initCurrentFast started from a given labeling, FastGCStereo.h:116-130) on the CPU emulator of the
kernel source: the designed scenes of tests/test_gpu_label_cost.py at emulator sizes, every pixel against the C oracle (cost-volume
energy), the numpy NaiveStereoEnergy oracle, and the compiled reference's own branch where oracle/_ref is built."""
import pytest

from emu import emu_lib
import label_cost_checks as LC


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
    with emu_lib.emulated():
        yield


@pytest.mark.parametrize("mode", [0, 1])
def test_emu_random_planes_both_views(mode):
    """Independent planes per pixel beyond both ends of [MIN, MAX], NaN and +-inf planes, a width that is not a multiple of 4."""
    LC.check_cost_volume_scene(19, 27, 9, 6, mode=mode)


def test_emu_generic_sampler_min_max():
    """MIN / MAX other than (0, D - 1): the generic sampler, whose slice index is shifted by -MIN."""
    LC.check_cost_volume_scene(17, 22, 12, 6, MIN=2.0, MAX=8.5, seed=1)


@pytest.mark.parametrize("windR", [4, 5, 7])
def test_emu_radii(windR):
    """windR odd and even: R = windR // 2 and windR >= 2R."""
    LC.check_cost_volume_scene(16, 21, 8, windR, seed=windR)


@pytest.mark.parametrize("H,W", [(6, 25), (25, 6), (1, 23), (23, 1), (3, 3)])
def test_emu_images_smaller_than_the_window(H, W):
    LC.check_cost_volume_scene(H, W, 7, 6, seed=H + W, nonfinite=0.0)


@pytest.mark.parametrize("mode", [0, 1])
def test_emu_naive_energy(mode):
    """The image-based energy: each pixel's warp comes from its own F(p); planes with v != 0."""
    LC.check_naive_scene(14, 19, 8, 7, mode=mode)   # odd windR: F(p) starts windR, the window 2R = windR - 1 left of p


def test_emu_argument_errors():
    LC.check_argument_errors()
