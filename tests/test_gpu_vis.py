"""The reference's debug images on the H100 (lexp_vis.cuh, DESIGN.md 3j): lexp_render_* against oracle/vis_oracle.py bit for bit on
designed states at 120 x 160 and on random-start states of both views at the benchmark's size (2048 x 1536 x 256), lexp_run_ex against
the composed run, and the command on the MiddV2 cones pair writing the reference's debug/ file set."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import run_checks as RC
import vis_checks as VC

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONES = os.path.join(ROOT, "tests", "golden", "middv2_cones")


@pytest.mark.parametrize("naive,min_disp", [(False, 0.0), (True, 0.0), (False, 2.5)])
def test_render_equals_the_oracle(naive, min_disp):
    E = VC.vis_energy(120, 160, 32, 20, naive=naive, min_disp=min_disp)
    try:
        VC.set_designed_state(E, (0, 1), seed=8)
        gt, nonocc = VC.designed_gt(E.height, E.width, E.MAX_DISPARITY, E.pm_get(0)[1], seed=8)
        assert VC.check_render_evaluation(E, gt, nonocc) == 6
        VC.check_render_consistency(E)
    finally:
        E.close()


def test_render_at_the_benchmark_size():
    """2048 x 1536 x 256 (the image-based energy, so no cost volume is needed): random starts of both views, then lexp_render_* of
    that state against the oracle."""
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import NativePMSweep
    from oracle import lexp_oracle as O
    H, W, D = 1536, 2048, 256
    prm = L.Parameters(windR=20, filterName="GF", filter_param1=1e-4)
    E = L.NaiveStereoEnergy(O.synthetic_image(H, W, 42), O.synthetic_image(H, W, 43), prm, D - 1)
    try:
        E.set_smoothness(**RC.SMOOTH)
        for m in (0, 1):
            S = NativePMSweep(E, unit_sizes=[25], proposers=[[(L.PROP_EXPANSION, 1)]], mode=m)
            try:
                S.begin()
                S.random_start(100 + m)
            finally:
                S.close()
        gt, nonocc = RC.synthetic_gt(E, 4)
        VC.check_render_evaluation(E, gt, nonocc, precisions=((-1.0, 0.5), (0.25, 0.5)))
        VC.check_render_consistency(E)
    finally:
        E.close()


def test_run_images_equal_the_composed_run():
    mk = lambda: RC.scene_energy(120, 160, 32, 20)
    VC.check_run_images(mk, (0, 1), 1, 1, [5, 15, 25], RC.PROPS + RC.PROPS[1:], seed=21)
    VC.check_run_images(mk, (0,), 1, 1, [5, 15, 25], RC.PROPS + RC.PROPS[1:], seed=22)
    mk = lambda: RC.scene_energy(120, 160, 32, 20, naive=True)
    VC.check_run_images(mk, (0, 1), 0, 1, [5, 15, 25], RC.PROPS + RC.PROPS[1:], seed=23)


def test_cli_writes_the_reference_debug_images_on_the_cones_pair(tmp_path):
    """-mode MiddV2 -doDual 1 -seed 7 (2 pm + 5 graph-cut iterations): debug/ holds exactly result{0,1}{D,N,E}00..08.png and
    result{0,1}C01..08.png, each decoded PNG equal to the oracle's image of the composed run's state at that point; disp0.pfm is the
    composed run's."""
    import cv2
    import localexpstereo_b200 as L
    from localexpstereo_b200 import cli
    out = tmp_path / "out"
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-m", "localexpstereo_b200", "-mode", "MiddV2", "-targetDir", CONES, "-outputDir", str(out),
                        "-doDual", "1", "-seed", "7"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=400)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0
    pngs = sorted(f for f in os.listdir(out / "debug") if f.endswith(".png"))
    dne = [f for f in pngs if re.fullmatch(r"result[01][DNE]\d\d\.png", f)]
    cc = [f for f in pngs if re.fullmatch(r"result[01]C\d\d\.png", f)]
    assert len(dne) == 54 and len(cc) == 16 and len(pngs) == 70
    assert sorted(dne) == sorted("result%d%s%02d.png" % (m, k, i) for i in range(9) for m in (0, 1) for k in "DNE")
    assert sorted(cc) == sorted("result%dC%02d.png" % (m, i) for i in range(1, 9) for m in (0, 1))
    o = cli.parse_args(["-mode", "MiddV2", "-targetDir", CONES])
    data = cli.load_data(CONES + "/")
    E, units, props, precision, threshold = cli.make_energy(o, data)
    try:
        want, lab, _ = VC.composed_run_images(E, (0, 1), 2, 5, units, props, 7, precision, threshold, data[2], data[3])
    finally:
        E.close()
    assert len(want) == 70
    for i, m, k, rendered, w in want:
        f = str(out / "debug" / ("result%d%s%02d.png" % (m, k, i)))
        got = cv2.imread(f, cv2.IMREAD_UNCHANGED)
        assert got is not None and got.shape == w.shape and np.array_equal(got, w), f
        assert np.array_equal(rendered, w), f
    L.save_pfm_file(str(tmp_path / "disp0.pfm"), cli.disparities(lab))
    assert (out / "disp0.pfm").read_bytes() == (tmp_path / "disp0.pfm").read_bytes()
    last = {k: w for i, m, k, _, w in want if i == 8 and m == 0}
    print("cones view 0 after the post-processing: E pixels 255 / 200 / 0 =", [int((last["E"] == v).sum()) for v in (255, 200, 0)])
    assert (last["E"] == 200).any() and (last["E"] == 0).any()
