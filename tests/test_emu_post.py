"""tests/test_gpu_post.py (post-processing of a two-view run: left-right check, dilation, hole filling, weighted median) on the CPU
emulator of the kernel source, bit for bit against the numpy oracle: the designed scenes, inf / NaN disparities under the x86-64
conversion rule, and a window radius larger than the image (every window clipped)."""
import numpy as np
import pytest

from emu import emu_lib
import test_gpu_post as _gp


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
    with emu_lib.emulated():
        yield


def test_emu_designed_scene_equals_the_oracle():
    H, W, windR = 20, 27, 4
    im0, im1, lab0, lab1 = _gp.designed_scene(H, W, seed=3)
    E = _gp.make_energy(im0, im1, windR)
    try:
        r = _gp.check_against_oracle(E, im0, im1, lab0, lab1, windR)
        f = r["fail"]
        assert f[0][1, 0] == 0 and f[0][2, 0] == 128 and f[1][1, W - 1] != 128 and (f[0][H - 3] == 128).all()
        assert (f == 255).any() and r["n_failed"] > 50
    finally:
        E.close()


def test_emu_nonfinite_disparities():
    H, W, windR = 16, 22, 3
    im0, im1, lab0, lab1 = _gp.designed_scene(H, W, seed=5, nonfinite=True)
    E = _gp.make_energy(im0, im1, windR)
    try:
        for thr in (1.5, 0.0):
            r = _gp.check_against_oracle(E, im0, im1, lab0, lab1, windR, threshold=thr)
            assert r["fail"][0][H // 2, W // 2] == 128 and r["fail"][0][0, 3] == 128
    finally:
        E.close()


def test_emu_every_window_clipped():
    H, W, windR = 10, 13, 16
    im0, im1, lab0, lab1 = _gp.designed_scene(H, W, seed=2)
    E = _gp.make_energy(im0, im1, windR, omega=25.0)
    try:
        _gp.check_against_oracle(E, im0, im1, lab0, lab1, windR, omega=25.0)
    finally:
        E.close()


def test_emu_error_paths():
    _gp.test_error_paths()
