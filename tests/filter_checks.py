"""Checks of the bilateral filter ("BL" / "BF") and the unfiltered mode ("") on the device (lexp_filters.cuh, DESIGN.md 3i), shared
by tests/test_emu_filters.py (CPU emulator) and tests/test_gpu_zz_filters.py (H100).

Every entry point is held against oracle/filter_oracle.py (FP64):
  * ""         bit for bit (the raw samplers restate the reference's float arithmetic exactly);
  * bilateral  |d| <= 1e-5 max(sum w |p|, 1e-3) -- the float rounding of the weights and of the window sum scale with sum w |p|;
  * the NaN and COST_FOR_INVALID patterns exactly.
The outputs of one call through every output path, two calls, and the warm start against the unary call (F(p), {p}) agree bit for
bit; a PatchMatch step is certified against its own unary instantiation: (P) proposals, (U) the update rule bit for bit with nothing
changing outside the targetRects, (Q) its costs against the oracle, (I) its costs equal the unary instantiation's."""
import ctypes as C

import numpy as np

import localexpstereo_b200 as L
from oracle import lexp_oracle as O
from oracle.filter_oracle import FilteredEnergyOracle
from label_cost_checks import device_costs, filter_rects, random_plane_field
from lexp_testlib import bits, make_scene

BL_REL = 1e-5
NAMES = {("cv", "bl"): "BL", ("cv", "none"): "", ("naive", "bl"): "BF", ("naive", "none"): ""}


def params(energy, filt, windR, sig2=10.0):
    name = NAMES[(energy, filt)]
    if energy == "naive":
        return L.Parameters(windR=windR, filterName=name, filter_param1=sig2)
    return L.Parameters(windR=windR, filterName=name, filter_param1=sig2, th_col=0.5)


def make_oracle(energy, filt, scene, windR, MIN, MAX, sig2=10.0):
    imL, imR, volL, volR = scene
    prm, bl = params(energy, filt, windR, sig2), filt == "bl"
    if energy == "naive":
        return FilteredEnergyOracle.naive(imL, imR, windR, sig2, prm.th_col, prm.th_grad, prm.alpha, MAX, MIN, bilateral=bl)
    return FilteredEnergyOracle.cost_volume(imL, imR, volL, volR, windR, sig2, prm.th_col, MAX, MIN, bilateral=bl)


def make(energy, filt, H, W, D, windR, seed=0, MIN=0.0, MAX=None, sig2=10.0, scene=None):
    """The context (E) and its oracle (Or) of CostVolumeEnergy (energy "cv") or NaiveStereoEnergy ("naive") with the bilateral
    filter (filt "bl") or none ("none")."""
    scene = make_scene(H, W, D, seed) if scene is None else scene
    imL, imR, volL, volR = scene
    MAX = float(D - 1 if MAX is None else MAX)
    prm = params(energy, filt, windR, sig2)
    if energy == "naive":
        E = L.NaiveStereoEnergy(imL, imR, prm, MAX, MIN)
    else:
        E = L.CostVolumeEnergy(imL, imR, volL, volR, prm, MAX, MIN)
    return E, make_oracle(energy, filt, scene, windR, MIN, MAX, sig2)


def compare(got, q, scale, exact, what=""):
    """Returns the worst |d| / max(sum w |p|, 1e-3) (0 for exact comparisons)."""
    got = np.asarray(got, np.float32)
    nan = np.isnan(q)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN pattern differs at {np.argwhere(np.isnan(got) != nan)[:5]}"
    assert np.array_equal(got == O.COST_FOR_INVALID, q == O.COST_FOR_INVALID), f"{what}: COST_FOR_INVALID mask differs"
    k = ~nan
    if exact:
        bad = bits(got[k]) != bits(q[k].astype(np.float32))
        assert not bad.any(), f"{what}: {int(bad.sum())} values differ, e.g. {got[k][bad][:3]} vs {q[k][bad][:3]}"
        return 0.0
    rel = np.abs(got[k].astype(np.float64) - q[k]) / np.maximum(scale[k], 1e-3)
    worst = float(rel.max()) if rel.size else 0.0
    assert worst <= BL_REL, f"{what}: worst |d| / sum w|p| = {worst:.3e}"
    return worst


def corner_calls(H, W, windR):
    """Calls with filterRects at every image corner, over the whole image and inside it (whose windows the filterRect, not the image,
    clips); disjoint targetRects of every shape (1x1, a sub-rect, the whole filterRect)."""
    fw, fh = min(W, 2 * windR + 3), min(H, 2 * windR + 2)
    f = [(0, 0, fw, fh), (W - fw, 0, fw, fh), (0, H - fh, fw, fh), (W - fw, H - fh, fw, fh), (0, 0, W, H), (W // 4, H // 4, W // 2, H // 2)]
    t = [(0, 0, 1, 1), (W - 3, 1, 3, 2), (1, H - 3, 4, 3), (W - 2, H - 1, 2, 1), (0, H // 2, 1, 1), (W // 4, H // 4, W // 2, H // 2)]
    return np.array(f, np.int32), np.array(t, np.int32)


def plan_planes(n, H, W, MIN, MAX, seed, v=False):
    """n planes: ordinary, steep, beyond [MIN, MAX], NaN / +-inf."""
    lab = random_plane_field(1, n, MIN, MAX, seed, v=v, slope=0.4).reshape(n, 4)
    lab[1 % n, 0] = np.float32(7.5)                   # steep
    if n > 3:
        lab[3, 2] = np.float32(np.nan)
    if n > 4:
        lab[4, 1] = np.float32(np.inf)
    return lab


def check_unary(dm, energy, filt, H, W, D, windR, mode=0, seed=0, MIN=0.0, MAX=None):
    """The unary calls of a plan against the oracle, with and without the check; image output (host and device), compact tiles
    (host and device) and a second call bit for bit."""
    E, Or = make(energy, filt, H, W, D, windR, seed, MIN, MAX)
    exact = filt == "none"
    worst = 0.0
    try:
        fr, tr = corner_calls(H, W, windR)
        planes = plan_planes(len(fr), H, W, E.MIN_DISPARITY, E.MAX_DISPARITY, 300 + seed, v=energy == "naive")
        P = E.make_plan(fr, tr)
        offs = np.concatenate([[0], np.cumsum(tr[:, 2] * tr[:, 3])])
        for wc in (True, False):
            img = np.full((H, W), -1.0, np.float32)
            P.eval_host(planes, img, with_check=wc, mode=mode)
            tiles = P.eval_host_tiles(planes, np.full(int(offs[-1]), -1.0, np.float32), with_check=wc, mode=mode)
            d_img = dm.zeros((H, W), -1.0)
            P.eval_device(planes, dm.ptr(d_img), W * 4, with_check=wc, mode=mode)
            d_tiles = dm.zeros((int(offs[-1]),), -1.0)
            P.eval_device_tiles(planes, dm.ptr(d_tiles), with_check=wc, mode=mode)
            E.sync()
            again = np.full((H, W), -1.0, np.float32)
            P.eval_host(planes, again, with_check=wc, mode=mode)
            assert np.array_equal(bits(img), bits(again)), "two calls differ"
            assert np.array_equal(bits(img), bits(dm.download(d_img))), "device image output differs from the host one"
            assert np.array_equal(bits(tiles), bits(dm.download(d_tiles))), "device tiles differ from host tiles"
            for i, (f, t) in enumerate(zip(fr, tr)):
                x, y, w, h = t
                got = img[y:y + h, x:x + w]
                assert np.array_equal(bits(got.ravel()), bits(tiles[offs[i]:offs[i + 1]])), f"call {i}: tiles differ from the image"
                q, scale = Or.unary(tuple(f), tuple(t), planes[i], mode, with_check=wc)
                worst = max(worst, compare(got, q, scale, exact, f"{energy}/{filt} call {i} check {wc}"))
        untouched = np.ones((H, W), bool)
        for x, y, w, h in tr:
            untouched[y:y + h, x:x + w] = False
        assert (img[untouched] == -1.0).all(), "a pixel outside the targetRects was written"
        P.close()
        return worst
    finally:
        E.close()


def check_warm_start(energy, filt, H, W, D, windR, mode=0, seed=0, MIN=0.0, MAX=None, unary_pixels=None, scene=None):
    """lexp_pm_init_from_labeling on independent random planes per pixel: the pixels `unary_pixels` (a seeded sample; all: None)
    against the oracle and bit for bit against the unary call (F(p), {p}) of the same plane.  scene: (imL, imR, volL, volR) in place
    of make_scene's (the view `mode`'s image and volume are required)."""
    E, Or = make(energy, filt, H, W, D, windR, seed, MIN, MAX, scene=scene)
    exact = filt == "none"
    try:
        lab = random_plane_field(H, W, E.MIN_DISPARITY, E.MAX_DISPARITY, 400 + seed, v=energy == "naive", nonfinite=0.02)
        got = device_costs(E, lab, mode)
        again = device_costs(E, lab, mode)
        assert np.array_equal(bits(got), bits(again)), "two calls differ"
        ys, xs = np.mgrid[0:H, 0:W]
        ys, xs = ys.ravel(), xs.ravel()
        if unary_pixels is not None:
            pick = np.random.default_rng(seed).choice(len(ys), size=min(unary_pixels, len(ys)), replace=False)
            ys, xs = ys[pick], xs[pick]
        F = filter_rects(H, W, windR, ys, xs)
        q = np.empty(len(ys))
        sc = np.empty(len(ys))
        for i, (y, x) in enumerate(zip(ys, xs)):
            a, b = Or.unary(tuple(F[i]), (int(x), int(y), 1, 1), lab[y, x], mode)
            q[i], sc[i] = a[0, 0], b[0, 0]
        worst = compare(got[ys, xs], q, sc, exact, f"warm start {energy}/{filt}")
        T = np.stack([xs, ys, np.ones_like(xs), np.ones_like(xs)], 1).astype(np.int32)
        P = E.make_plan(F, T)
        tiles = P.eval_host_tiles(lab[ys, xs], np.empty(len(ys), np.float32), with_check=True, mode=mode)
        P.close()
        assert np.array_equal(bits(tiles), bits(got[ys, xs])), "warm start differs from the unary call (F(p), {p})"
        return worst
    finally:
        E.close()


def check_pm_steps(dm, energy, filt, H, W, D, windR, unit, mode=0, seed=0, MIN=0.0, MAX=None, sig2=10.0, layer_group=0):
    """One group of a layer: an initialisation step, then a step of every proposer kind (list, Expansion, Random, RANSAC), each
    certified (P)(U)(Q)(I) against the device's own pre-step state."""
    E, Or = make(energy, filt, H, W, D, windR, seed, MIN, MAX, sig2)
    exact = filt == "none"
    worst = 0.0
    try:
        lm = L.LayerManager(W, H, windR)
        ly = lm.addLayer(unit)
        cells = ly.disjointRegionSets[layer_group]
        units = np.array([ly.unitRegions[i] for i in cells], np.int32)
        tr = np.array([ly.sharedRegions[i] for i in cells], np.int32)
        fr = np.array([ly.filterRegions[i] for i in cells], np.int32)
        P = E.make_plan(fr, tr)
        P.set_units(units)
        n = len(cells)
        inside = np.zeros((H, W), bool)
        for x, y, w, h in tr:
            inside[y:y + h, x:x + w] = True
        rng = O.CvRNG(seed + 1)
        init_planes = np.stack([O.create_random_label(rng, u[0] + u[2] // 2, u[1] + u[3] // 2, E.MIN_DISPARITY, E.MAX_DISPARITY) for u in units])
        E.pm_begin(mode, None, random_plane_field(H, W, E.MIN_DISPARITY, E.MAX_DISPARITY, 500 + seed))
        d_out = dm.zeros((n, 4))
        steps = [(L.PROP_LIST, 0, init_planes, True), (L.PROP_LIST, 0, plan_planes(n, H, W, E.MIN_DISPARITY, E.MAX_DISPARITY, 600 + seed), False),
                 (L.PROP_EXPANSION, 0, None, False), (L.PROP_RANDOM, 1, None, False), (L.PROP_RANSAC, 0, None, False),
                 (L.PROP_RANDOM, 4, None, False)]
        for k, (kind, m, planes, init) in enumerate(steps):
            pre_c, pre_l = E.pm_get(mode)
            s = 1000 + 17 * k + seed
            P.pm_step(0, kind, m, s, planes=planes, d_planes_out=dm.ptr(d_out), init=init, mode=mode)
            post_c, post_l = E.pm_get(mode)
            used = np.asarray(dm.download(d_out), np.float32).reshape(n, 4)
            # (P) proposals on the pre-step state
            if kind == L.PROP_LIST:
                assert np.array_equal(bits(used), bits(planes))
            else:
                want = np.stack([O.pm_proposal(kind, m, O.pm_rng_state(s, i), pre_l, tuple(int(v) for v in u), E.MIN_DISPARITY, E.MAX_DISPARITY) for i, u in enumerate(units)])
                if kind == L.PROP_RANDOM:
                    assert np.array_equal(bits(used[:, 3]), bits(want[:, 3])) and np.allclose(used, want, rtol=2e-6, atol=1e-6)
                else:
                    assert np.array_equal(bits(used), bits(want)), f"step {k}: proposals differ"
            # (I) the unary instantiation of the same planes
            q_img = np.full((H, W), np.nan, np.float32)
            P.eval_host(used, q_img, with_check=True, mode=mode)
            # (U) the update rule, nothing outside the targetRects
            upd = inside & (True if init else (pre_c > q_img))
            want_c = np.where(upd, q_img, pre_c)
            want_l = pre_l.copy()
            for i, (x, y, w, h) in enumerate(tr):
                sl = (slice(y, y + h), slice(x, x + w))
                want_l[sl][upd[sl]] = used[i]
            assert np.array_equal(bits(post_c), bits(want_c)), f"step {k}: costs differ from the update rule"
            assert np.array_equal(bits(post_l), bits(want_l)), f"step {k}: labels differ from the update rule"
            # (Q) the step's costs against the oracle
            for i, (f, t) in enumerate(zip(fr, tr)):
                x, y, w, h = t
                q, scale = Or.unary(tuple(f), tuple(t), used[i], mode)
                worst = max(worst, compare(q_img[y:y + h, x:x + w], q, scale, exact, f"step {k} call {i}"))
        P.close()
        return worst
    finally:
        E.close()


def check_errors(energy, filt):
    """A context without the guided filter refuses peer wiring and enqueues nothing; sig2 <= 0 / non-finite is refused."""
    import pytest
    E, _ = make(energy, filt, 12, 16, 6, 4)
    try:
        E.pm_begin(0)
        n0 = E.launch_count
        with pytest.raises(L.LexpError, match="guided filter only"):
            peers = (C.c_void_p * 1)(E._h.value)
            L._capi.check(L._capi.lib().lexp_pm_connect_local(E._h, 0, 0, 1, C.cast(peers, C.c_void_p)))
        assert E.launch_count == n0
    finally:
        E.close()
    if filt == "bl":
        for bad in (0.0, -1.0, float("inf"), float("nan")):
            with pytest.raises(L.LexpError, match="sig2"):
                make(energy, filt, 12, 16, 6, 4, sig2=bad)


def cones_scene(D=20, seed=5):
    """The cones crop (tests/golden/cones_crop_d20.npz: the MiddV2 cones images, 128 x 160) with a synthetic volume."""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cones_crop_d20.npz"))
    imL, imR = g["imL"], g["imR"]
    H, W = imL.shape[:2]
    return imL, imR, O.synthetic_volume(D, H, W, 1234 + seed), O.synthetic_volume(D, H, W, 1235 + seed)


def check_against_reference(energy, filt, H, W, D, windR, mode=0, seed=0, MIN=0.0, MAX=None, scene=None, device=False):
    """The compiled reference's own energy with this filterName (oracle/_ref/liblexp_ref_filters.so) on the corner calls, with and
    without the check: the FP64 oracle against it (cost-volume "" bit for bit, image-based "" within 1e-4 relative, bilateral within
    1e-5 sum w |p|) -- and with device=True the device's costs under the same rules.  Returns the worst relative error."""
    from oracle.ref_filters import RefFilterEnergy
    from lexp_testlib import assert_costs_close
    scene = make_scene(H, W, D, seed) if scene is None else scene
    imL, imR, volL, volR = scene
    H, W = imL.shape[:2]
    MAX = float(D - 1 if MAX is None else MAX)
    E = make(energy, filt, H, W, D, windR, seed, MIN, MAX, scene=scene)[0] if device else None
    Or = make_oracle(energy, filt, scene, windR, MIN, MAX)
    prm = params(energy, filt, windR)
    R = RefFilterEnergy(0 if energy == "cv" else 1, imL, imR, volL, volR, windR, NAMES[(energy, filt)], prm.filter_param1, prm.th_col,
                        prm.th_grad, prm.alpha, MAX, MIN)
    worst = 0.0
    try:
        fr, tr = corner_calls(H, W, windR)
        planes = plan_planes(len(fr), H, W, MIN, MAX, 700 + seed, v=energy == "naive")
        P = E.make_plan(fr, tr) if device else None
        for wc in (True, False):
            img = None
            if device:
                img = np.full((H, W), -1.0, np.float32)
                P.eval_host(planes, img, with_check=wc, mode=mode)
            for i, (f, t) in enumerate(zip(fr, tr)):
                ref = R.unary(f, t, planes[i], mode, wc)
                q, scale = Or.unary(tuple(f), tuple(t), planes[i], mode, with_check=wc)
                x, y, w, h = t
                for what, got in (("oracle", q), ("device", None if img is None else img[y:y + h, x:x + w])):
                    if got is None:
                        continue
                    tag = f"{what} vs reference {energy}/{filt} windR {windR} mode {mode} call {i} check {wc}"
                    got = np.asarray(got, np.float64)
                    assert np.array_equal(np.isnan(got), np.isnan(ref)), tag + ": NaN pattern"
                    k = ~np.isnan(ref)
                    if filt == "none" and energy == "cv":
                        assert np.array_equal(bits(got[k].astype(np.float32)), bits(ref[k])), tag
                    elif filt == "none":
                        worst = max(worst, assert_costs_close(got[k].astype(np.float32), ref[k], tag))
                    else:
                        assert np.array_equal(got[k] == O.COST_FOR_INVALID, ref[k] == O.COST_FOR_INVALID), tag + ": invalid mask"
                        rel = np.abs(got[k] - ref[k].astype(np.float64)) / np.maximum(scale[k], 1e-3)
                        worst = max(worst, float(rel.max()) if rel.size else 0.0)
                        assert worst <= BL_REL, f"{tag}: worst |d| / sum w|p| = {worst:.3e}"
        if P is not None:
            P.close()
        return worst
    finally:
        R.close()
        if E is not None:
            E.close()
