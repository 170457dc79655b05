"""The PatchMatch phase of the image-based energy (NaiveStereoEnergy, `-mode MiddV2`) on the device, step by step against the
oracle's update of the SAME state (tests/pm_step_rig.py with naive=True: (Q) on a sample of each step's cells, no pixel tags):
scenes shared by tests/test_gpu_zz_naive_pm.py and tests/test_emu_naive_pm.py.
A whole-run replay would drift at the exact FP32 ties of the truncated image cost (tests/test_gpu_zz_gc.py explains them); a
per-step certification does not."""
import numpy as np

from oracle import lexp_oracle as O
from lexp_testlib import seeded_labels
from pm_step_rig import Rig, run_sweep

MIDDV2_LAMBDA = 20.0   # main.cpp:72 paramsGF
MIDDV2_UNITS = [5, 15, 25]   # main.cpp:304-306


def cones(H=None, W=None):
    """The natural-image crop of data/MiddV2/cones the golden vectors use (128 x 160), optionally cut to H x W."""
    import lexp_golden
    G = lexp_golden.load()
    imL, imR = G["imL"], G["imR"]
    return np.ascontiguousarray(imL[:H, :W]), np.ascontiguousarray(imR[:H, :W])


def middv2_params(windR=20, lam=MIDDV2_LAMBDA):
    import localexpstereo_b200 as L
    return L.Parameters(lambda_=lam, windR=windR, filterName="GF", filter_param1=1e-4)   # th_col 10, th_grad 2, alpha 0.9


def with_v(labels, seed):
    """The same planes with a nonzero fourth component (a vertical offset of the warp, StereoEnergy.h:720-725) per unit."""
    out = np.array(labels, np.float32)
    out[:, 3] = np.random.default_rng(seed).choice(np.float32([-1.5, -0.75, 0.5, 1.25]), len(out))
    return out


def naive_rig(devmem, imL, imR, D, windR, units, proposers, mode=0, q_cells=4, seed=0):
    """The step rig on the image-based energy with MiddV2's parameters at windR, disparities 0 .. D - 1."""
    return Rig(devmem, imL, imR, None, None, windR, units, proposers, mode, MAX=D - 1, naive=True, q_cells=q_cells, seed=seed)


# ---- scenes --------------------------------------------------------------------------------------------------------------------------------
def reference_lists(n_layers):
    from localexpstereo_b200.sweep import V3_PROPOSERS_REFERENCE
    return V3_PROPOSERS_REFERENCE[:n_layers]


def scene_cones(devmem, mode, H=None, W=None, units=None, iterations=2, seed=3):
    """The cones crop at windR 20 with the reference's proposer lists (RANSAC included) and MiddV2's layers."""
    imL, imR = cones(H, W)
    units = units or MIDDV2_UNITS
    R = naive_rig(devmem, imL, imR, 64, 20, units, reference_lists(len(units)), mode, seed=seed)
    try:
        T = run_sweep(R, seeded_labels(R.S, 40 + seed), iterations, 500 + seed, what=f"cones crop {R.H} x {R.W}, windR 20, mode {mode}")
        assert T.n_exact > 50 and T.n_random > 50
        return T
    finally:
        R.close()


def scene_generic_radius(devmem, mode=0, H=61, W=83, iterations=2):
    """windR 12: the generic-radius instantiation <0, true, true>, on a ragged synthetic pair."""
    import localexpstereo_b200 as L
    imL, imR = O.synthetic_image(H, W, 52), O.synthetic_image(H, W, 53)
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANSAC, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]]
    R = naive_rig(devmem, imL, imR, 24, 12, [7, 19], props, mode, seed=1)
    try:
        T = run_sweep(R, seeded_labels(R.S, 11), iterations, 77, what=f"synthetic {H} x {W}, windR 12, mode {mode}")
        assert T.n_exact > 50 and T.n_random > 50
        return T
    finally:
        R.close()


def scene_vertical_offset(devmem, mode=1, H=72, W=96):
    """Planes with v != 0 (the proposers copy v): the warp shifted vertically, on the cones crop."""
    import localexpstereo_b200 as L
    imL, imR = cones(H, W)
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]]
    R = naive_rig(devmem, imL, imR, 32, 20, [5, 15], props, mode, seed=2)
    try:
        labels = with_v(seeded_labels(R.S, 9), 9)
        T = run_sweep(R, labels, 1, 31, what=f"v != 0, cones crop {H} x {W}, mode {mode}")
        lab = R.S.get()[1]
        assert (lab[..., 3] != 0).all()
        return T
    finally:
        R.close()
