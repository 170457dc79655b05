"""The reference's debug images (lexp_vis.cuh, DESIGN.md 3j) on the CPU emulator of the kernel source: lexp_render_* against
oracle/vis_oracle.py bit for bit on designed states of both energies and both views, and lexp_run_ex's images at exactly the reference's
points, each equal to the composed run's at that point."""
import numpy as np
import pytest

from emu import emu_lib
import run_checks as RC
import vis_checks as VC


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
    import os
    prev = os.environ.get("LEXP_GC_THREADS")
    os.environ["LEXP_GC_THREADS"] = "128"
    with emu_lib.emulated():
        yield
    if prev is None:
        os.environ.pop("LEXP_GC_THREADS", None)
    else:
        os.environ["LEXP_GC_THREADS"] = prev


@pytest.mark.parametrize("naive,min_disp", [(False, 0.0), (True, 0.0), (False, 2.5)])
def test_emu_render_equals_the_oracle(naive, min_disp):
    E = VC.vis_energy(36, 52, 12, 6, naive=naive, min_disp=min_disp)
    try:
        VC.set_designed_state(E, (0, 1), seed=5)
        gt, nonocc = VC.designed_gt(E.height, E.width, E.MAX_DISPARITY, E.pm_get(0)[1], seed=5)
        assert VC.check_render_evaluation(E, gt, nonocc) == 6
        c0, c1 = VC.check_render_consistency(E)
        assert (c0[..., 0] == 255).any() and (c0[..., 2] == 255).any()   # both kinds of failure occur
        d, n, e = E.render_evaluation(0, -1.0, 0.5)
        assert set(np.unique(e)) == {0, 200, 255}
        # a = b = 0: G = R = (0 * 1 + 1) / 2 * 255 = 127.5, rounded to even
        flat = (E.pm_get(0)[1][..., :2] == 0).all(axis=-1)
        assert (n[flat][:, 1:] == 128).all() and (n[flat][:, 0] == 255).all()
        # ground truth without a valid value, a mask of zeros: every E pixel 255 (no GT) and then every wrong one 200
        E.set_ground_truth(np.full_like(gt, np.inf), np.zeros_like(nonocc))
        assert (E.render_evaluation(1, 0.25, 0.5)[2] == 255).all()
        VC.check_render_evaluation(E, gt, np.zeros_like(nonocc), modes=(1,), precisions=((0.25, 0.5),))
    finally:
        E.close()


def test_emu_render_needs_its_state():
    from localexpstereo_b200._capi import LexpError
    E = RC.scene_energy(24, 32, 8, 6)
    try:
        E.pm_begin(0)
        with pytest.raises(LexpError, match="ground_truth"):
            E.render_evaluation(0)
        gt, nonocc = RC.synthetic_gt(E, 1)
        E.set_ground_truth(gt, nonocc)
        with pytest.raises(LexpError, match="lexp_pm_begin"):
            E.render_evaluation(1)
        with pytest.raises(LexpError, match="lexp_pm_begin"):
            E.render_consistency()
    finally:
        E.close()


def test_emu_run_images_need_ground_truth():
    from localexpstereo_b200._capi import LexpError
    E = RC.scene_energy(24, 32, 8, 6)
    try:
        n = E.launch_count
        with pytest.raises(LexpError, match="ground_truth"):
            E.run(1, (0,), 0, None, [8], RC.PROPS[:1], 3, image_callback=lambda *a: None)
        assert E.launch_count == n
    finally:
        E.close()


@pytest.mark.parametrize("naive,views,pm", [(False, (0,), 1), (False, (0, 1), 1), (False, (0, 1), 0), (True, (0, 1), 1)])
def test_emu_run_images_equal_the_composed_run(naive, views, pm):
    mk = lambda: RC.scene_energy(32, 48, 10, 6, naive=naive)
    imgs = VC.check_run_images(mk, views, pm, 1, [8, 16], RC.PROPS, seed=11)
    assert len(imgs) == len(VC.expected_images(views, pm, 1))


def test_emu_run_image_callback_errors_are_reraised():
    E = RC.scene_energy(24, 32, 8, 6)
    try:
        gt, nonocc = RC.synthetic_gt(E, 2)
        E.set_ground_truth(gt, nonocc)
        seen = []

        def boom(i, m, k, a):
            seen.append((i, m, k))
            raise KeyError("image")
        with pytest.raises(KeyError):
            E.run(1, (0,), 0, None, [8], RC.PROPS[:1], 3, image_callback=boom)
        assert seen == VC.expected_images((0,), 0, 1)
    finally:
        E.close()
