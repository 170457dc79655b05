"""-mode MiddV3 of the command on the CPU emulator: a synthetic im0.acrt and no im1.acrt, so the right view's volume is derived from the left
file (LEXP_VOL_RIGHT_FROM_LEFT), layers v3_layer_units(width), precision -1 and the error threshold of the directory name.  The output must
equal the same run composed from the public calls on volumes uploaded from memory with the same preparation."""
import os

import numpy as np
import pytest

from emu import emu_lib
import run_checks as RC
from lexp_testlib import make_scene


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
    with emu_lib.emulated():
        yield


def test_emu_middv3_with_a_synthetic_acrt_and_no_im1(tmp_path, capsys):
    import cv2
    import localexpstereo_b200 as L
    from localexpstereo_b200 import cli
    from localexpstereo_b200.sweep import V3_PROPOSERS_REFERENCE, v3_layer_units
    H, W, D = 24, 200, 8
    imL, imR, volL, _ = make_scene(H, W, D, seed=3)
    d = tmp_path / "trainingQ" / "Pair"
    d.mkdir(parents=True)
    cv2.imwrite(str(d / "im0.png"), imL); cv2.imwrite(str(d / "im1.png"), imR)
    with open(d / "calib.txt", "w") as f:
        f.write(f"width={W}\nheight={H}\nndisp={D}\n")
    volL.astype(np.float32).tofile(str(d / "im0.acrt"))   # raw float[D][H][W], no header
    gt = np.random.default_rng(1).uniform(1, D - 1, (H, W)).astype(np.float32)
    with open(d / "disp0GT.pfm", "wb") as f:
        f.write(f"Pf\n{W} {H}\n-1.000000\n".encode() + np.ascontiguousarray(gt[::-1]).astype("<f4").tobytes())
    out = tmp_path / "out"
    o = cli.parse_args(["-mode", "MiddV3", "-targetDir", str(d), "-outputDir", str(out), "-doDual", "1", "-iterations", "0",
                        "-pmIterations", "0", "-filterRadious", "4", "-seed", "5"])
    assert o["smooth_weight"] == 0.5 and cli.error_threshold_v3(str(d)) == 0.5
    rows = cli.run(o)
    assert "im1.acrt not found" in capsys.readouterr().out
    lines = (out / "debug" / "log_output.txt").read_text().splitlines()
    assert len(lines) == 3 and len(rows) == 2 and float((out / "time.txt").read_text()) >= 0
    prm = L.Parameters(lambda_=0.5, windR=4, filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.CostVolumeEnergy(imL, imR, None, None, prm, D - 1)
    try:
        E.set_volume(0, volL, L.VOL_FILL)
        E.set_volume(1, volL, L.VOL_RIGHT_FROM_LEFT)
        E.set_smoothness(0.5, prm.omega, prm.th_smooth, prm.epsilon)
        E.set_ground_truth(gt, None)
        lab, raw, pts = RC.composed_run(E, (0, 1), 0, 0, v3_layer_units(W), V3_PROPOSERS_REFERENCE, 5, None, -1.0, 0.5)
    finally:
        E.close()
    for name, labeling in (("disp0.pfm", lab), ("disp0raw.pfm", raw)):
        L.save_pfm_file(str(tmp_path / name), cli.disparities(labeling))
        assert (out / name).read_bytes() == (tmp_path / name).read_bytes(), name
    mine = [e for i, m, e in pts if m == 0]
    for line, e in zip(lines[1:], mine):
        assert line.split("\t")[1:] == ["%f" % e[k] for k in ("energy", "data", "smooth", "all", "nonocc")]
