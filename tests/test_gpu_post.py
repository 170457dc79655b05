"""Post-processing of a two-view run on the device (lexp_post_process = PMStereoBase::postProcess, PMStereoBase.h:146-256): the left-right
check, the dilation, the hole filling and the weighted median, against the numpy oracle (tests/post_oracle.py) BIT FOR BIT -- fail maps,
both final labelings, and currentCost_ untouched -- and, on the cones crop after a device two-view run, against the reference's own
postProcess compiled in oracle/_ref (when that library is present): labelings bit-identical except at pixels where the chosen median key
is tied (the order std::sort gives equal keys is unspecified), where the disparity is still bit-identical; disp0.pfm byte-identical.

The scenes are shared with tests/test_emu_post.py (the same kernels on the CPU emulator).  On the 2048 x 1536 scenes the oracle's median
runs on a random sample of the failed pixels (the fail maps and every other pixel are compared in full)."""
import ctypes as C

import numpy as np
import pytest

import post_oracle as P
from lexp_testlib import bits, seeded_labels

pytestmark = pytest.mark.gpu

OMEGA = 10.0


def make_energy(im0, im1, windR, omega=OMEGA, smooth=True):
    import localexpstereo_b200 as L
    E = L.CostVolumeEnergy(im0, im1, None, None, L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5), 63)
    if smooth:
        E.set_smoothness(1.0, omega, 1.0, 0.01)
    return E


# ---- scenes -----------------------------------------------------------------------------------------------------------------------
def blocky_image(H, W, rng, block=5):
    """8-bit BGR image of random colour blocks plus a little noise: many equal and many different weights"""
    base = rng.integers(0, 256, ((H + block - 1) // block, (W + block - 1) // block, 3))
    im = np.repeat(np.repeat(base, block, 0), block, 1)[:H, :W]
    return np.clip(im + rng.integers(-3, 4, (H, W, 3)), 0, 255).astype(np.uint8)


def fronto(c, v=0.0):
    return np.array([0.0, 0.0, c, v], np.float32)


def designed_scene(H, W, seed=0, nonfinite=False):
    """Both views of a foreground box (disparity 6) over a background (disparity 2), consistent except for the occlusion bands
    (width 4) beside the box, the invisible bands at the left border of view 0 / right border of view 1, a fully failed row, random
    outliers, slanted patches, hole-fill ties (equal GetZ from both sides) and the rx cases x - d + 0.5 = -0.4 (inside: truncation
    toward zero), -1.1 (outside) and W - 0.1 (inside).  nonfinite: also +-inf and NaN disparities (the device's NaN rule)."""
    rng = np.random.default_rng(seed)
    D0, D1 = 2.0, 6.0
    lab0 = np.tile(fronto(D0), (H, W, 1))
    lab1 = lab0.copy()
    bx0, bx1, by0, by1 = W // 3, W // 3 + W // 4, H // 4, H // 4 + H // 3
    lab0[by0:by1, bx0:bx1] = fronto(D1, 1.0)
    lab1[by0:by1, bx0 - int(D1):bx1 - int(D1)] = fronto(D1, 1.0)
    n = max(1, H * W // 30)                                            # outliers in both views
    for lab in (lab0, lab1):
        ys, xs = rng.integers(0, H, n), rng.integers(0, W, n)
        lab[ys, xs, 2] = rng.uniform(0.0, 12.0, n).astype(np.float32)
        lab[ys, xs, 3] = rng.integers(2, 9, n).astype(np.float32)
    sy, sx = min(H - 4, 3 * H // 4), min(W - 8, 2 * W // 3)            # slanted patch (consistent in neither view)
    lab0[sy:sy + 3, sx:sx + 6, 0] = np.float32(0.25)
    lab0[sy:sy + 3, sx:sx + 6, 2] = np.float32(D0 - 0.25 * sx)
    lab0[H - 3, :] = fronto(1e6)                                       # a fully failed row (every rx outside)
    ty = 2 if H > 8 else 0                                             # hole-fill tie: equal GetZ on both sides of a failed run
    lab0[ty, W // 2 - 3] = fronto(D0, 5.0)
    lab0[ty, W // 2 - 2:W // 2 + 2] = fronto(40.0)
    lab0[ty, W // 2 + 2] = fronto(D0, 7.0)
    lab0[1, 0] = fronto(0.9)                                           # v = -0.4 -> rx = 0, inside
    lab0[2 % H, 0] = fronto(1.6)                                       # v = -1.1 -> outside
    lab1[1, W - 1] = fronto(0.4)                                       # v = W - 0.1 -> rx = W - 1, inside
    if nonfinite:
        lab0[0, 3] = fronto(np.inf); lab0[H - 1, W - 2] = fronto(-np.inf)
        lab1[H // 2, 1] = fronto(np.inf)
        lab0[H // 2, W // 2] = fronto(np.nan); lab1[1, 1] = fronto(np.nan)
        lab0[H // 2 + 1, 2] = np.array([np.inf, 0.0, 1.0, 0.0], np.float32)   # inf * 0 = NaN keys in windows that hold it
    im0, im1 = blocky_image(H, W, rng), blocky_image(H, W, rng)
    return im0, im1, lab0, lab1


def random_scene(H, W, frac, seed=0):
    """Consistent fronto-parallel planes whose disparity varies with y only (b != 0), with a fraction `frac` of the pixels of each view
    replaced by random planes: about 2 * frac of the pixels fail, plus the invisible bands at the borders."""
    rng = np.random.default_rng(seed)
    lab = np.zeros((H, W, 4), np.float32)
    lab[..., 1] = np.float32(0.01)
    lab[..., 2] = np.float32(8.0)
    labs = []
    for _ in range(2):
        l = lab.copy()
        m = rng.random((H, W)) < frac
        k = int(m.sum())
        l[m] = np.stack([rng.uniform(-0.2, 0.2, k), rng.uniform(-0.2, 0.2, k), rng.uniform(0, 40, k), rng.integers(0, 4, k)], 1).astype(np.float32)
        labs.append(l)
    return blocky_image(H, W, rng, 7), blocky_image(H, W, rng, 7), labs[0], labs[1]


# ---- device run and oracle comparison ----------------------------------------------------------------------------------------------
def run_device(E, lab0, lab1, threshold=1.5):
    H, W = lab0.shape[:2]
    costs = [np.full((H, W), 3.5, np.float32), np.arange(H * W, dtype=np.float32).reshape(H, W)]
    E.pm_begin(0, costs[0], lab0)
    E.pm_begin(1, costs[1], lab1)
    fail = np.zeros((2, H, W), np.uint8)
    E.post_process(threshold, fail)
    c0, o0 = E.pm_get(0)
    c1, o1 = E.pm_get(1)
    assert np.array_equal(bits(c0), bits(costs[0])) and np.array_equal(bits(c1), bits(costs[1])), "currentCost_ was touched"
    return o0, o1, fail


def sample_failed(fail, n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(2):
        ys, xs = np.nonzero(fail[i] > 0)
        if len(ys) <= n:
            out.append(list(zip(ys, xs)))
            continue
        pick = np.unique(np.concatenate([[0, len(ys) - 1], rng.choice(len(ys), n, replace=False)]))
        out.append(list(zip(ys[pick], xs[pick])))
    return out


def check_against_oracle(E, im0, im1, lab0, lab1, windR, omega=OMEGA, threshold=1.5, sample=None, seed=0):
    got0, got1, fail = run_device(E, lab0, lab1, threshold)
    pixels = None if sample is None else sample_failed(P.consistency_check(lab0, lab1, threshold), sample, seed)
    want0, want1, fail_o, tied, done = P.post_process(lab0, lab1, im0, im1, windR, omega, threshold, pixels)
    assert np.array_equal(fail, fail_o), f"fail maps differ at {np.argwhere(fail != fail_o)[:5].tolist()}"
    for i, (got, want, lab) in enumerate(((got0, want0, lab0), (got1, want1, lab1))):
        keep = fail[i] == 0
        assert np.array_equal(bits(got[keep]), bits(lab[keep])), f"view {i}: a consistent pixel changed"
        d = done[i]
        bad = np.argwhere(d & (bits(got) != bits(want)).any(axis=2))
        assert len(bad) == 0, f"view {i}: {len(bad)} of {int(d.sum())} median pixels differ, first {bad[:3].tolist()}: " \
                              f"{got[tuple(bad[0])]} vs {want[tuple(bad[0])]}"
    return dict(got=(got0, got1), fail=fail, n_failed=int((fail > 0).sum()), n_checked=int(done[0].sum() + done[1].sum()), tied=tied)


# ---- reference (oracle/_ref/liblexp_ref_post.so, built where the reference sources are) -------------------------------------------
def ref_lib():
    from oracle import build_ref_post
    path = build_ref_post.build()
    if path is None:
        return None
    L = C.CDLL(path)
    L.ref_post_create.restype = C.c_void_p
    L.ref_post_create.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_float]
    L.ref_post_destroy.argtypes = [C.c_void_p]
    L.ref_post_process.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int]
    L.ref_consistency_check.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p]
    L.ref_post_last_error.restype = C.c_char_p
    L.ref_post_save_pfm.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int]
    return L


def ref_post_process(R, im0, im1, lab0, lab1, windR, omega=OMEGA, threshold=1.5, nthreads=0):
    """The reference's postProcess and doConsistencyCheck: (out0, out1, fail)"""
    H, W = lab0.shape[:2]
    h = R.ref_post_create(H, W, np.ascontiguousarray(im0).ctypes.data, np.ascontiguousarray(im1).ctypes.data, windR, omega, 64.0)
    assert h, R.ref_post_last_error()
    try:
        d0, d1 = P.disparities(lab0), P.disparities(lab1)
        fail = np.zeros((2, H, W), np.uint8)
        assert R.ref_consistency_check(h, d0.ctypes.data, d1.ctypes.data, H, W, threshold, fail.ctypes.data) == 0, R.ref_post_last_error()
        o0, o1 = np.ascontiguousarray(lab0.copy()), np.ascontiguousarray(lab1.copy())
        assert R.ref_post_process(h, o0.ctypes.data, o1.ctypes.data, H, W, threshold, nthreads) == 0, R.ref_post_last_error()
        return o0, o1, fail
    finally:
        R.ref_post_destroy(h)


def check_against_reference(got0, got1, fail, tied, ref):
    """Bit-identical labelings except at tied median keys, where the disparity is bit-identical."""
    r0, r1, rfail = ref
    assert np.array_equal(np.where(rfail > 0, rfail, 0), fail)
    n_tied = 0
    for i, (got, want) in enumerate(((got0, r0), (got1, r1))):
        diff = (bits(got) != bits(want)).any(axis=2)
        assert not (diff & ~tied[i]).any(), f"view {i}: {int((diff & ~tied[i]).sum())} pixels differ outside key ties"
        assert np.array_equal(bits(P.disparities(got))[diff], bits(P.disparities(want))[diff])
        n_tied += int(diff.sum())
    return n_tied


# ---- tests ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W,windR", [(48, 64, 4), (37, 53, 12)])
def test_designed_scene_equals_the_oracle(H, W, windR):
    im0, im1, lab0, lab1 = designed_scene(H, W, seed=H)
    E = make_energy(im0, im1, windR)
    try:
        r = check_against_oracle(E, im0, im1, lab0, lab1, windR)
        f = r["fail"]
        assert f[0][1, 0] == 0 and f[0][2 % H, 0] == 128 and f[1][1, W - 1] != 128     # rx = trunc(-0.4) = 0 and trunc(W - 0.1) = W - 1
        assert (f[0][H - 3] == 128).all()                                               # the fully failed row
        assert (f[0][:, 0] == 128).any() and (f[1][:, W - 1] == 128).any() and (f[0] == 255).any() and (f[1] == 255).any()
    finally:
        E.close()


def test_nonfinite_disparities_and_thresholds():
    """inf / NaN disparities: NaN and |v| >= 2^31 are "outside" (128) as x86-64's conversion makes them; NaN keys sort last"""
    H, W, windR = 30, 41, 6
    im0, im1, lab0, lab1 = designed_scene(H, W, seed=5, nonfinite=True)
    E = make_energy(im0, im1, windR)
    try:
        for thr in (1.5, 0.0, 7.0):
            r = check_against_oracle(E, im0, im1, lab0, lab1, windR, threshold=thr)
            assert r["fail"][0][H // 2, W // 2] == 128 and r["fail"][0][0, 3] == 128
    finally:
        E.close()


def test_every_window_clipped():
    """windR larger than the image: every window is clipped on all sides"""
    H, W, windR = 18, 21, 24
    im0, im1, lab0, lab1 = designed_scene(H, W, seed=2)
    E = make_energy(im0, im1, windR, omega=25.0)
    try:
        check_against_oracle(E, im0, im1, lab0, lab1, windR, omega=25.0)
    finally:
        E.close()


@pytest.mark.parametrize("frac,lo,hi", [(0.025, 0.03, 0.08), (0.17, 0.25, 0.36)])
def test_2048x1536_r20(frac, lo, hi):
    """The default workload's size at windR 20 (1 681 candidates) with about 5 % and about 30 % failed pixels"""
    H, W, windR = 1536, 2048, 20
    im0, im1, lab0, lab1 = random_scene(H, W, frac, seed=int(frac * 1000))
    E = make_energy(im0, im1, windR)
    try:
        r = check_against_oracle(E, im0, im1, lab0, lab1, windR, sample=1500, seed=1)
        assert lo < r["n_failed"] / (2 * H * W) < hi, r["n_failed"] / (2 * H * W)
        if frac > 0.1:   # two calls from the same snapshot
            again = run_device(E, lab0, lab1)
            assert np.array_equal(bits(again[0]), bits(r["got"][0])) and np.array_equal(bits(again[1]), bits(r["got"][1]))
            assert np.array_equal(again[2], r["fail"])
        else:            # on a caller's stream
            import torch
            s = torch.cuda.Stream()
            E.set_stream(s.cuda_stream)
            again = run_device(E, lab0, lab1)
            torch.cuda.synchronize()
            assert np.array_equal(bits(again[0]), bits(r["got"][0])) and np.array_equal(bits(again[1]), bits(r["got"][1]))
    finally:
        E.close()


def test_windR_32_and_a_ragged_size():
    """windR 32 (4 225 candidates, 64 KB of sort entries) and 437 x 291 at windR 20"""
    for (H, W, windR, frac) in ((300, 412, 32, 0.05), (291, 437, 20, 0.08)):
        im0, im1, lab0, lab1 = random_scene(H, W, frac, seed=W)
        E = make_energy(im0, im1, windR)
        try:
            check_against_oracle(E, im0, im1, lab0, lab1, windR, sample=1200, seed=2)
        finally:
            E.close()


def cones_two_view_state():
    """Both views of the cones crop after a device two-view run: initialisation, one pm iteration and one graph-cut iteration per view"""
    import lexp_golden
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import GCSweep
    G = lexp_golden.load()
    H, W = G["imL"].shape[:2]
    prm = L.Parameters(windR=G["windR"], filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.CostVolumeEnergy(G["imL"], G["imR"], G["volL"], G["volR"], prm, G["D"] - 1)
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 2)], [(L.PROP_EXPANSION, 1)]]
    labs = []
    for mode in (0, 1):
        S = GCSweep(E, unit_sizes=[6, 18, 40], proposers=props, mode=mode, lam=1.0, omega=OMEGA, th_smooth=1.0, epsilon=0.01)
        S.begin()
        S.init(seeded_labels(S, 31 + mode))
        S.iteration(0, 500 + mode)
        S.gc_iteration(0, 600 + mode)
        labs.append(E.pm_get(mode)[1])
    return E, G, labs


def test_cones_crop_after_a_device_two_view_run(tmp_path):
    E, G, (lab0, lab1) = cones_two_view_state()
    try:
        im0, im1, windR = G["imL"], G["imR"], G["windR"]
        raw = E.computeDisparities(0)
        assert np.array_equal(bits(raw), bits(P.disparities(lab0)))
        r = check_against_oracle(E, im0, im1, lab0, lab1, windR)
        assert r["n_failed"] > 100
        out = E.computeDisparities(0)
        from localexpstereo_b200.energy import save_pfm_file
        save_pfm_file(str(tmp_path / "disp0.pfm"), out)
        R = ref_lib()
        if R is None:
            pytest.skip("oracle/_ref/liblexp_ref_post.so is not built on this machine (it needs the reference sources)")
        ref = ref_post_process(R, im0, im1, lab0, lab1, windR)
        check_against_reference(*r["got"], r["fail"], r["tied"], ref)
        # disp0.pfm from the reference's postProcess output, written by the reference's own save_pfm_file
        d_ref = np.ascontiguousarray(P.disparities(ref[0]))
        assert R.ref_post_save_pfm(str(tmp_path / "ref_disp0.pfm").encode(), d_ref.ctypes.data, d_ref.shape[0], d_ref.shape[1]) == 0
        assert (tmp_path / "disp0.pfm").read_bytes() == (tmp_path / "ref_disp0.pfm").read_bytes()
    finally:
        E.close()


def test_error_paths():
    import localexpstereo_b200 as L
    H, W = 20, 24
    im0, im1, lab0, lab1 = designed_scene(H, W)
    E = make_energy(im0, im1, 4, smooth=False)
    try:
        E.pm_begin(0, None, lab0)
        with pytest.raises(L.LexpError, match="error -3"):   # view 1 has no state
            E.post_process()
        E.pm_begin(1, None, lab1)
        with pytest.raises(L.LexpError, match="lexp_set_smoothness"):
            E.post_process()
        E.set_smoothness(1.0, OMEGA, 1.0, 0.01)
        E.post_process()
    finally:
        E.close()
