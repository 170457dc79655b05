"""The oracle of the post-processing (tests/post_oracle.py) against the reference's own PMStereoBase::doConsistencyCheck and postProcess
(PMStereoBase.h:111-256), compiled from its headers into oracle/_ref/liblexp_ref_post.so (oracle/build_ref_post.py).  Fail maps must be
identical; labelings bit-identical except at pixels where the oracle's chosen median key is tied with another candidate's (std::sort
leaves their order unspecified), and there the disparity must still be bit-identical.  No scene here has a NaN median key (undefined
behaviour of the reference's comparator)."""
import numpy as np
import pytest

import post_oracle as P
import test_gpu_post as _gp

R = _gp.ref_lib()
if R is None:
    pytest.skip("oracle/_ref/liblexp_ref_post.so is not built and the reference's headers are absent", allow_module_level=True)


def pin(im0, im1, lab0, lab1, windR, omega=_gp.OMEGA, threshold=1.5):
    ref = _gp.ref_post_process(R, im0, im1, lab0, lab1, windR, omega, threshold)
    o0, o1, fail, tied, done = P.post_process(lab0, lab1, im0, im1, windR, omega, threshold)
    assert np.array_equal(fail, ref[2]), f"fail maps differ at {np.argwhere(fail != ref[2])[:5].tolist()}"
    n_tied = _gp.check_against_reference(o0, o1, fail, tied, ref)
    return dict(fail=fail, n_failed=int((fail > 0).sum()), n_tied_diff=n_tied, n_tied=int(tied[0].sum() + tied[1].sum()))


@pytest.mark.parametrize("H,W,windR,omega", [(48, 64, 4, 10.0), (37, 53, 12, 10.0), (18, 21, 24, 25.0), (60, 80, 20, 3.0)])
def test_designed_scenes(H, W, windR, omega):
    """Occlusion bands beside a box in both views, invisible bands at the borders, a fully failed row, outliers, slanted patches,
    hole-fill ties, rx on -0.4 / -1.1 / W - 0.1; the (18, 21, 24) case clips every window"""
    im0, im1, lab0, lab1 = _gp.designed_scene(H, W, seed=H)
    r = pin(im0, im1, lab0, lab1, windR, omega)
    f = r["fail"]
    assert f[0][1, 0] == 0 and f[0][2, 0] == 128 and f[1][1, W - 1] != 128 and (f[0][H - 3] == 128).all()
    assert (f[0][:, 0] == 128).any() and (f[1][:, W - 1] == 128).any() and (f == 255).any()


def test_infinite_disparities():
    """+-inf disparities (keys +-inf, never NaN): outside (128) in the check, ordered like numbers in the median"""
    H, W, windR = 30, 41, 6
    im0, im1, lab0, lab1 = _gp.designed_scene(H, W, seed=5)
    lab0[0, 3] = _gp.fronto(np.inf); lab0[H - 1, W - 2] = _gp.fronto(-np.inf); lab1[H // 2, 1] = _gp.fronto(np.inf)
    for thr in (1.5, 0.0, 7.0):
        r = pin(im0, im1, lab0, lab1, windR, threshold=thr)
        assert r["fail"][0][0, 3] == 128 and r["fail"][0][H - 1, W - 2] == 128


def test_occlusion_band_widths():
    """A box of disparity 6 over a background of 2: in view 0 the 4 pixels left of the box see a background point that view 1 covers by
    the box (255); at x = 0 the matched point is outside the image (128), at x = 1 rx = int(-0.5) = 0 is inside"""
    H, W = 24, 40
    lab0 = np.tile(_gp.fronto(2.0), (H, W, 1)); lab1 = lab0.copy()
    lab0[6:18, 16:26] = _gp.fronto(6.0); lab1[6:18, 10:20] = _gp.fronto(6.0)
    rng = np.random.default_rng(0)
    im0, im1 = _gp.blocky_image(H, W, rng), _gp.blocky_image(H, W, rng)
    f = pin(im0, im1, lab0, lab1, 5)["fail"]
    assert f[0][10, 0] == 128 and (f[0][10, 1:12] == 0).all() and (f[0][10, 12:16] == 255).all() and (f[0][10, 16:] == 0).all()
    assert (f[1][10, W - 2:] == 128).all() and f[1][10, W - 3] == 0 and (f[1][10, 20:24] == 255).all()


def test_cones_crop():
    """The natural images of the cones crop with a piecewise-planar two-view state: 4 x 4 blocks of random planes around a smooth
    disparity, consistent between the views where the planes agree"""
    import lexp_golden
    from oracle import lexp_oracle as O
    G = lexp_golden.load()
    H, W = G["imL"].shape[:2]
    rng = O.CvRNG(9)
    labs = []
    for mode in (0, 1):
        lab = np.tile(_gp.fronto(6.0), (H, W, 1))
        for y in range(0, H, 4):
            for x in range(0, W, 4):
                if (x * 7 + y * 3 + mode) % 5 == 0:
                    lab[y:y + 4, x:x + 4] = O.create_random_label(rng, x, y, 0.0, G["D"] - 1.0)
        labs.append(lab)
    r = pin(G["imL"], G["imR"], labs[0], labs[1], G["windR"])
    assert r["n_failed"] > 500
