"""The command's debug images (cli.imwrite through lexp_run_ex) on the CPU emulator: -mode MiddV3 -doDual 1 on a synthetic pair writes
the reference's debug/ file set, each PNG decoding to the composed run's image at that point, and the other outputs stay as they were.
The PIL fallback of cli.imwrite writes the same pixels as cv2."""
import builtins
import os

import numpy as np
import pytest

from emu import emu_lib
import run_checks as RC
import vis_checks as VC
from lexp_testlib import make_scene


@pytest.fixture(scope="module", autouse=True)
def _use_emulator():
    with emu_lib.emulated():
        yield


def test_emu_cli_writes_the_debug_images(tmp_path):
    import cv2
    import localexpstereo_b200 as L
    from localexpstereo_b200 import cli
    from localexpstereo_b200.sweep import V3_PROPOSERS_REFERENCE, v3_layer_units
    H, W, D = 24, 200, 8
    imL, imR, volL, volR = make_scene(H, W, D, seed=4)
    d = tmp_path / "trainingQ" / "Pair"
    d.mkdir(parents=True)
    cv2.imwrite(str(d / "im0.png"), imL); cv2.imwrite(str(d / "im1.png"), imR)
    with open(d / "calib.txt", "w") as f:
        f.write(f"width={W}\nheight={H}\nndisp={D}\n")
    volL.astype(np.float32).tofile(str(d / "im0.acrt"))
    volR.astype(np.float32).tofile(str(d / "im1.acrt"))
    gt = np.random.default_rng(2).uniform(1, D - 1, (H, W)).astype(np.float32)
    with open(d / "disp0GT.pfm", "wb") as f:
        f.write(f"Pf\n{W} {H}\n-1.000000\n".encode() + np.ascontiguousarray(gt[::-1]).astype("<f4").tobytes())
    out = tmp_path / "out"
    o = cli.parse_args(["-mode", "MiddV3", "-targetDir", str(d), "-outputDir", str(out), "-doDual", "1", "-iterations", "0",
                        "-pmIterations", "0", "-filterRadious", "4", "-seed", "5"])
    rows = cli.run(o)
    assert len(rows) == 2
    pngs = sorted(f for f in os.listdir(out / "debug") if f.endswith(".png"))
    assert pngs == sorted(["result%d%s%02d.png" % (m, k, i) for i in range(2) for m in (0, 1) for k in "DNE"] +
                          ["result%dC01.png" % m for m in (0, 1)])
    prm = L.Parameters(lambda_=0.5, windR=4, filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.CostVolumeEnergy(imL, imR, None, None, prm, D - 1)
    try:
        E.set_volume(0, volL, L.VOL_FILL)
        E.set_volume(1, volR, L.VOL_FILL)
        E.set_smoothness(0.5, prm.omega, prm.th_smooth, prm.epsilon)
        E.set_ground_truth(gt, None)
        want, lab, raw = VC.composed_run_images(E, (0, 1), 0, 0, v3_layer_units(W), V3_PROPOSERS_REFERENCE, 5, -1.0, 0.5, gt, None)
    finally:
        E.close()
    assert len(want) == len(pngs)
    for i, m, k, rendered, w in want:
        got = cv2.imread(str(out / "debug" / ("result%d%s%02d.png" % (m, k, i))), cv2.IMREAD_UNCHANGED)
        assert np.array_equal(got, w) and np.array_equal(rendered, w), (i, m, k)
    for name, labeling in (("disp0.pfm", lab), ("disp0raw.pfm", raw)):
        L.save_pfm_file(str(tmp_path / name), cli.disparities(labeling))
        assert (out / name).read_bytes() == (tmp_path / name).read_bytes(), name


def test_imwrite_without_cv2_writes_the_same_pixels(tmp_path, monkeypatch):
    import cv2
    from localexpstereo_b200 import cli
    rng = np.random.default_rng(0)
    gray = rng.integers(0, 256, (13, 17), dtype=np.uint8)
    bgr = rng.integers(0, 256, (13, 17, 3), dtype=np.uint8)
    real_import = builtins.__import__

    def no_cv2(name, *a, **k):
        if name == "cv2":
            raise ImportError("cv2 hidden")
        return real_import(name, *a, **k)
    monkeypatch.setattr(builtins, "__import__", no_cv2)
    cli.imwrite(str(tmp_path / "g.png"), gray)
    cli.imwrite(str(tmp_path / "c.png"), bgr)
    monkeypatch.setattr(builtins, "__import__", real_import)
    assert np.array_equal(cv2.imread(str(tmp_path / "g.png"), cv2.IMREAD_UNCHANGED), gray)
    assert np.array_equal(cv2.imread(str(tmp_path / "c.png"), cv2.IMREAD_UNCHANGED), bgr)
