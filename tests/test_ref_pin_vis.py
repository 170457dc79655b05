"""The debug-image oracle (oracle/vis_oracle.py) against the reference's own code (oracle/_ref/liblexp_ref_vis.so: the real
Evaluator::evaluate and viewConsistencyCheck, their images captured at cv::imwrite), on designed states: disparities on k + 0.5 after
scaling and one ulp either side, negative ones and ones above max_disp, NaN / inf planes, a = b = 0, GT 0 and inf, occluded wrong
pixels, precision -1 / a power of two / the cones pair's gt_prec / another, MIN_DISPARITY != 0 for the C images, both views.  And
vis_oracle.sat8, imwrite's conversion of a float image to 8 bits, against cv2 where it is importable.

The one allowed difference: the shim evaluates disparityMapVis = disp * F / 255 eagerly, as two float roundings (* F, then / 255), where
OpenCV 3.1 folds it into one convertTo with scale F * (1 / 255).  The oracle (and the device) follow OpenCV.  A D pixel may therefore
differ by one grey level where both chains land within a few ulp of a half-integer, and only there; the test prints how many do."""
import numpy as np
import pytest

from oracle import lexp_oracle as O
from oracle import ref_vis
from oracle import vis_oracle as V
import vis_checks as VC

if not ref_vis.available():
    pytest.skip("oracle/_ref/liblexp_ref_vis.so is not built and the reference's headers are absent", allow_module_level=True)

H, W = 36, 52
IM_L = O.synthetic_image(H, W, 5)
IM_R = O.synthetic_image(H, W, 6)
CONES_GT_PREC = float(np.float32(1.0) / np.float32(4))   # loadData: 1.0f / gt_scale with the cones pair's info.txt


def _d_levels_agree(mine, ref, what):
    """sat8 of the oracle's float D against sat8 of the reference's: equal, except one level apart where the oracle's value lies within
    4 ulp of the half-integer between the two levels (and the reference's on the other side of it).  Returns the count of such pixels."""
    a, b = V.sat8(mine).astype(int), V.sat8(ref).astype(int)
    diff = np.argwhere(a != b)
    for y, x in diff:
        assert abs(a[y, x] - b[y, x]) == 1, (what, y, x, mine[y, x], ref[y, x])
        mid = np.float32(min(a[y, x], b[y, x]) + 0.5)
        ulp = np.spacing(mid)
        assert abs(mine[y, x] - mid) <= 4 * ulp and abs(ref[y, x] - mid) <= 4 * ulp, (what, y, x, mine[y, x], ref[y, x])
    return len(diff)


@pytest.mark.parametrize("max_disp", [15.0, 58.0, 255.0])
def test_evaluator_images_equal_the_reference(max_disp):
    near = 0
    for mode in (0, 1):
        lab = VC.designed_labeling(H, W, max_disp, seed=int(max_disp) + mode)
        gt, nonocc = VC.designed_gt(H, W, max_disp, lab, seed=int(max_disp) + 2 * mode)
        for precision, threshold in ((-1.0, 0.5), (0.5, 0.5), (CONES_GT_PREC, 0.5), (0.3, 1.0)):
            d_ref, n_ref, e_ref = ref_vis.evaluate_images(IM_L, IM_R, max_disp, lab, gt, nonocc, precision, threshold, mode)
            what = (max_disp, mode, precision)
            assert np.array_equal(V.e_image(lab, gt, nonocc, precision, threshold), e_ref), what
            assert set(np.unique(e_ref)) == {0, 200, 255}, what
            n = V.n_float(lab)
            assert np.array_equal(n.view(np.uint32), n_ref.view(np.uint32)) or np.array_equal(n, n_ref, equal_nan=True), what
            near += _d_levels_agree(V.d_float(lab, precision, max_disp), d_ref, what)
            d, nn, e = V.eval_images(lab, gt, nonocc, precision, threshold, max_disp)
            assert np.array_equal(nn, V.sat8(n_ref)) and np.array_equal(e, e_ref)
    flat = (lab[..., :2] == 0).all(axis=-1)
    assert (V.sat8(V.n_float(lab))[flat][:, 1:] == 128).all()   # a = b = 0: 127.5 -> 128
    print(f"max_disp {max_disp}: {near} D pixels one grey level apart at a half-integer (the shim's two roundings of disp * F / 255)")


@pytest.mark.parametrize("min_disp,max_disp", [(0.0, 15.0), (2.5, 58.0), (-3.0, 40.0)])
def test_consistency_images_equal_the_reference(min_disp, max_disp):
    lab0 = VC.designed_labeling(H, W, max_disp, seed=3)
    lab1 = VC.designed_labeling(H, W, max_disp, seed=4)
    lab1[::2] = lab0[::2]   # half the rows consistent where the disparity is 0 there
    want = ref_vis.check_images(IM_L, IM_R, min_disp, max_disp, lab0, lab1)
    got = V.check_images(lab0, lab1, min_disp, max_disp)
    for m in range(2):
        assert np.array_equal(got[m], want[m]), (m, np.argwhere(got[m] != want[m])[:5])
        assert (want[m][..., 0] == 255).any() and (want[m][..., 2] == 255).any()


def test_sat8_equals_imwrite_of_a_float_image(tmp_path):
    """imwrite's conversion of a float image to 8 bits (cvRound, then saturation) in cv2: ties to even, saturation, NaN and values
    outside int32 to 0."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    special = np.array([0.5, 1.5, 2.5, 127.5, 128.5, 254.5, 255.5, 300, -3, -0.5, -0.6, np.nan, np.inf, -np.inf, 2147483520.0,
                        2147483648.0, -2147483648.0, 3e9, -3e9, 1e-45, 255.49998, 0.49999997], np.float32)
    vals = np.concatenate([special, rng.uniform(-20, 280, 4000).astype(np.float32),
                           (rng.integers(-2, 258, 2000) + np.float32(0.5)).astype(np.float32)])
    img = np.resize(vals, (60, 101)).astype(np.float32)
    for ch in (1, 3):
        a = img if ch == 1 else np.stack([img, img[::-1], img[:, ::-1]], axis=-1)
        path = str(tmp_path / f"f{ch}.png")
        assert cv2.imwrite(path, a)
        back = cv2.imread(path, cv2.IMREAD_UNCHANGED)
        assert np.array_equal(back, V.sat8(a)), np.argwhere(back != V.sat8(a))[:5]
