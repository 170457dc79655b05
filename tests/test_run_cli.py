"""The command `python -m localexpstereo_b200` on the host: ArgsParser's rules and the Options defaults, and every fallback of loadData
(main.cpp:201-268).  The run itself is in tests/test_gpu_zz_run.py."""
import os

import numpy as np
import pytest

from localexpstereo_b200 import cli

CONES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "middv2_cones")


def test_parse_args_defaults_per_mode():
    o = cli.parse_args(["-mode", "MiddV2", "-targetDir", "a", "-outputDir", "b"])
    assert (o["smooth_weight"], o["iterations"], o["pmIterations"], o["doDual"], o["filterRadious"], o["mc_threshold"], o["seed"]) == \
        (1.0, 5, 2, False, 20, 0.5, 0)
    assert cli.parse_args(["-mode", "MiddV3"])["smooth_weight"] == 0.5
    assert cli.parse_args(["-smooth_weight", "0.3", "-mode", "MiddV3"])["smooth_weight"] == 0.3   # an explicit value wins in any order
    assert cli.parse_args([])["smooth_weight"] == 1.0


@pytest.mark.parametrize("s,want", [("true", True), ("false", False), ("1", True), ("0", False), ("2", True), ("-1", True), ("0x", False)])
def test_parse_args_booleans(s, want):
    assert cli.parse_args(["-doDual", s])["doDual"] is want


def test_parse_args_pairs_and_numbers():
    o = cli.parse_args(["prog", "-iterations", "3", "-pmIterations", "0", "-ndisp", "64", "-seed", "9", "-trailing"])
    assert (o["iterations"], o["pmIterations"], o["ndisp"], o["seed"]) == (3, 0, 64, 9)
    assert cli.parse_args(["-iterations", " 7abc"])["iterations"] == 7   # std::stoi reads the leading integer
    with pytest.raises(ValueError):
        cli.parse_args(["-iterations", "x"])


def test_cv2_and_pil_decode_the_fixture_alike(monkeypatch):
    cv = {n: cli.imread(os.path.join(CONES, n), gray=g) for n, g in (("imL.png", False), ("groundtruth.png", True), ("nonocc.png", True))}
    import builtins
    real = builtins.__import__
    monkeypatch.setattr(builtins, "__import__", lambda name, *a, **k: (_ for _ in ()).throw(ImportError()) if name == "cv2" else real(name, *a, **k))
    for n, g in (("imL.png", False), ("groundtruth.png", True), ("nonocc.png", True)):
        pil = cli.imread(os.path.join(CONES, n), gray=g)
        assert pil.dtype == cv[n].dtype and np.array_equal(pil, cv[n]), n
    assert cv["imL.png"].shape == (375, 450, 3)


def test_load_data_cones():
    imL, imR, gt, nonocc, ndisp, prec = cli.load_data(CONES + "/")
    assert ndisp == 59 and prec == 0.25 and imL.shape == imR.shape == (375, 450, 3)
    g = cli.imread(os.path.join(CONES, "groundtruth.png"), gray=True)
    assert np.array_equal(np.isinf(gt), g == 0) and np.array_equal(gt[g > 0], g[g > 0].astype(np.float32) / 4)
    assert set(np.unique(nonocc)) <= {0, 255}


def test_load_data_fallbacks(tmp_path):
    d = str(tmp_path) + "/"
    imL = cli.imread(os.path.join(CONES, "imL.png"))[:40, :60]
    import cv2
    assert cli.load_data(d) is None                                   # no ndisp anywhere
    with open(d + "calib.txt", "w") as f:
        f.write("cam0=[1 0 0; 0 1 0; 0 0 1]\nwidth=60\nndisp=32\nisint=0\n")
    assert cli.load_data(d) is None                                   # no images
    cv2.imwrite(d + "im0.png", imL); cv2.imwrite(d + "im1.png", imL[:, ::-1].copy())
    im0, im1, gt, nonocc, ndisp, prec = cli.load_data(d)
    assert ndisp == 32 and prec < 0 and np.array_equal(im0, imL)
    assert (gt == 0).all() and (nonocc == 255).all()                  # no ground truth, no mask
    assert cli.load_data(d, ndisp=48)[4] == 48                        # -ndisp wins over calib.txt
    want = np.random.default_rng(0).uniform(1, 30, (40, 60)).astype(np.float32)
    with open(d + "disp0GT.pfm", "wb") as f:   # save_pfm_file's layout: rows bottom-up, little-endian floats
        f.write(b"Pf\n60 40\n-0.003922\n" + np.ascontiguousarray(want[::-1]).astype("<f4").tobytes())
    m = np.random.default_rng(1).choice(np.array([0, 128, 255], np.uint8), (40, 60))
    cv2.imwrite(d + "mask0nocc.png", m)
    _, _, gt, nonocc, _, _ = cli.load_data(d)
    assert np.array_equal(gt, want) and np.array_equal(nonocc, np.where(m == 255, 255, 0))
    cv2.imwrite(d + "nonocc.png", 255 - m)                            # nonocc.png before mask0nocc.png
    assert np.array_equal(cli.load_data(d)[3], np.where(m == 0, 255, 0))
    with open(d + "info.txt", "w") as f:                              # info.txt before calib.txt; groundtruth.png before the pfm
        f.write("8\n20\n")
    g = np.random.default_rng(2).integers(0, 200, (40, 60)).astype(np.uint8)
    cv2.imwrite(d + "groundtruth.png", g)
    cv2.imwrite(d + "imL.png", imL[:, ::-1].copy()); cv2.imwrite(d + "imR.png", imL)
    im0, _, gt, _, ndisp, prec = cli.load_data(d)
    assert ndisp == 20 and prec == 0.125 and np.array_equal(im0, imL[:, ::-1])
    assert np.array_equal(np.isinf(gt), g == 0) and np.array_equal(gt[g > 0], g[g > 0].astype(np.float32) / 8)


def test_error_threshold_of_middv3():
    assert [cli.error_threshold_v3(p) for p in ("a/trainingQ/x", "b/testF/y", "c/trainingH/z")] == [0.5, 2.0, 1.0]


def test_host_disparities_match_the_oracle():
    from oracle import run_oracle as RO
    lab = np.random.default_rng(3).normal(0, 3, (30, 40, 4)).astype(np.float32)
    assert np.array_equal(cli.disparities(lab).view(np.uint32), RO.disparities(lab).view(np.uint32))
