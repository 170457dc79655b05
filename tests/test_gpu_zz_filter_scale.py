"""The bilateral filter ("BL" / "BF") and the unfiltered mode ("") at the benchmark's size and in the right view (DESIGN.md 3i): whole
PatchMatch sweeps with every step certified by tests/pm_step_rig.py -- (P) the proposal, (U) the update rule bit for bit with nothing
changing outside the targetRects, (Q) the proposal costs against the FP64 oracle under the rules of tests/filter_checks.compare, (I)
the PatchMatch costs equal the unary instantiation's -- and the final state equal to the twin's uninterrupted sweep bit for bit:
  * bench.py's workload (2048 x 1536 x 256, windR 20), iteration 0, "BL" with V3_PROPOSERS_DEVICE and "" with V3_PROPOSERS_REFERENCE
    (RANSAC included): the initialisation and every step of layer 2 certified, the steps of layers 0 and 1 issued one by one; (Q)
    on every target pixel (the C oracle);
  * sampled unary cells of all three layers at that size through eval_host and eval_device_tiles, and the warm start;
  * the right view at 960 x 544 x 96, windR 32, "BL", two iterations;
  * the image-based energy with paramsBF on the MiddV2 cones pair, both views, (Q) on sampled cells.
The scene functions also run on the CPU emulator at small sizes (tests/test_emu_filter_sweeps.py).
(Sorted after the other filter tests and before the large-size tests.)"""
import os
import time

import numpy as np
import pytest

from lexp_testlib import TorchDeviceMemory, bits, make_scene, seeded_labels
from pm_step_rig import Rig, run_sweep

pytestmark = pytest.mark.gpu

SIG2 = 10.0
CONES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "middv2_cones")


@pytest.fixture(scope="module")
def devmem():
    return TorchDeviceMemory()


# ---- scenes, shared with the emulator ----------------------------------------------------------------------------------------------------
def scene_filter_sweep(devmem, energy, filt, mode, H, W, D, windR, units, proposers, iterations=1, seed=0, q_cells=4, layers=None):
    """A synthetic pair, the sweep under test step by step with every step (of `layers`, None: all) certified, the final state against
    the twin.  energy "cv" (filt "BL" / "") or "naive" (filt "BF" / "")."""
    imL, imR, volL, volR = make_scene(H, W, D, seed=seed)
    naive = energy == "naive"
    R = Rig(devmem, imL, imR, None if naive else volL, None if naive else volR, windR, units, proposers, mode,
            MAX=D - 1 if naive else None, naive=naive, q_cells=q_cells, seed=seed, filter=filt, sig2=SIG2)
    try:
        t0 = time.perf_counter()
        T = run_sweep(R, seeded_labels(R.S, 30 + seed), iterations, 700 + seed, layers=layers,
                      what=f"{energy} {filt!r} {W} x {H} x {D}, windR {windR}, mode {mode}, layers {layers or 'all'} certified")
        print(f"  {time.perf_counter() - t0:.1f} s in all")
        return T
    finally:
        R.close()


def scene_cones_bf(devmem, mode, units=(5, 15, 25), iterations=1, crop=None, q_cells=4, layers=None):
    """-mode MiddV2 with paramsBF (Parameters(lambda, windR 20, "BF", 10)) on the MiddV2 cones pair (crop: its top-left h x w),
    V3_PROPOSERS_REFERENCE, the initialisation and every step of `layers` (None: all) certified, (Q) on q_cells cells per step."""
    from localexpstereo_b200 import cli
    from localexpstereo_b200.sweep import V3_PROPOSERS_REFERENCE
    imL, imR, gt, nonocc, ndisp, prec = cli.load_data(CONES + "/")
    if crop is not None:
        imL, imR = [np.ascontiguousarray(im[:crop[0], :crop[1]]) for im in (imL, imR)]
    R = Rig(devmem, imL, imR, None, None, 20, list(units), V3_PROPOSERS_REFERENCE[:len(units)], mode, MAX=ndisp - 1, naive=True,
            q_cells=q_cells, seed=mode, filter="BF", sig2=SIG2)
    try:
        t0 = time.perf_counter()
        T = run_sweep(R, seeded_labels(R.S, 50 + mode), iterations, 900 + mode, layers=layers,
                      what=f"cones {R.W} x {R.H} paramsBF, layers {list(units)}, mode {mode}, layers {layers or 'all'} certified")
        print(f"  {time.perf_counter() - t0:.1f} s in all")
        assert T.ransac > 0 and T.q_cells >= T.steps
        return T
    finally:
        R.close()


# ---- the benchmark's workload ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bench_scene():
    """bench.py's PatchMatch-phase workload, as tests/test_gpu_zz_pm_steps.py's bench_rig builds it: 2048 x 1536 x 256, windR 20, the
    guide of bench.py, the volume drawn on the device (torch.rand, seed 1234) and copied to the host for the oracles (3.2 GB)."""
    import torch
    from localexpstereo_b200 import synth
    W, H, D, windR = 2048, 1536, 256, 20
    imL = synth.synthetic_image(H, W, 42)
    vol = torch.rand((D, H, W), generator=torch.Generator(device="cuda").manual_seed(1234), device="cuda", dtype=torch.float32)
    torch.cuda.synchronize()
    yield imL, vol, vol.cpu().numpy(), windR
    del vol
    torch.cuda.empty_cache()


BENCH_SEED = 4321


@pytest.mark.parametrize("filt,props,layers", [("BL", "device", (2,)), ("", "reference", (2,))])
def test_every_step_of_the_benchmark_workload(devmem, bench_scene, filt, props, layers):
    """The initialisation and every step of iteration 0 in `layers` certified, the other steps issued one by one uncertified;
    bench.py's initial labels (seed 99), the state tagged after the initialisation on both contexts; the state at the end of the
    iteration equals the twin's uninterrupted sweep bit for bit.  Layer 2 only: certifying a step at this size takes seconds
    on the host (the FP64 bilateral oracle, the proposal oracle of a layer-0 group's ~490 cells), too slow for all 241 in one test."""
    import torch
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import V3_PROPOSERS_DEVICE, V3_PROPOSERS_REFERENCE
    from pm_step_rig import assert_same_state
    imL, vol, vol_host, windR = bench_scene
    t0 = time.perf_counter()
    R = Rig(devmem, imL, None, vol, None, windR, None, V3_PROPOSERS_DEVICE if props == "device" else V3_PROPOSERS_REFERENCE,
            vol_host=vol_host, filter=filt, sig2=SIG2)
    try:
        units = R.S.lm.layers[0].unitRegions
        labels = synth.synthetic_planes([units[i] for i in range(len(units))], 1, vol.shape[0], 99)[0][R.S.init_index]
        ref = R.twin_reference(labels, BENCH_SEED, (0, 2), tag=True)
        R.E.pm_begin(0)
        R.init(labels)
        R.tag(R.E)
        R.iteration(0, BENCH_SEED, certify=lambda g: g.layer in layers)
        what = f"benchmark workload {filt!r}, V3_PROPOSERS_{props.upper()}, iteration 0, layers {list(layers)} certified"
        assert_same_state(R.get(R.E), ref, what)
        print(R.T.line(what) + f"; {time.perf_counter() - t0:.1f} s in all")
        assert R.T.steps == 1 + 16 * sum((9, 3, 3)[li] for li in layers)
        if props == "reference":
            assert R.T.ransac > 0
    finally:
        R.close()
        torch.cuda.empty_cache()


def _c_oracle(img, vol_host, windR, D):
    from oracle import c_oracle
    H, W = img.shape[:2]
    C = c_oracle.COracle(H, W, D, windR, 1e-4, 0.5, D - 1)
    C.set_image(0, img)
    C.set_volume(0, vol_host)
    return C


def test_sampled_unary_cells_of_every_layer(devmem, bench_scene):
    """Both filters at the benchmark's size: the last (border) group and a random group of each layer through eval_host and
    eval_device_tiles (bit-identical), sampled cells -- always the largest filterRect and the cell reaching furthest right and down --
    against the C oracle on their whole targetRects."""
    import localexpstereo_b200 as L
    import filter_checks as FC
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import v3_layer_units
    imL, vol, vol_host, windR = bench_scene
    D, (H, W) = int(vol.shape[0]), imL.shape[:2]
    C = _c_oracle(imL, vol_host, windR, D)
    t0 = time.perf_counter()
    try:
        for filt in ("BL", ""):
            E = L.CostVolumeEnergy(imL, None, vol, None, L.Parameters(windR=windR, filterName=filt, filter_param1=SIG2, th_col=0.5), D - 1)
            rng = np.random.default_rng(23)
            worst, n_cells, n_px, corner_layers = 0.0, 0, 0, set()
            try:
                lm = L.LayerManager(W, H, windR)
                for li, u in enumerate(v3_layer_units(W)):
                    lay = lm.addLayer(u)
                    ng = len(lay.disjointRegionSets)
                    corner = [r for r, (x, y, w, h) in enumerate(lay.sharedRegions) if (x + w, y + h) == (W, H)]
                    g_corner = [g for g in range(ng) if corner[0] in lay.disjointRegionSets[g]]
                    for gi in sorted({ng - 1, int(rng.integers(ng - 1))} | set(g_corner)):
                        grp = lay.disjointRegionSets[gi]
                        planes = synth.synthetic_planes(lay.unitRegions, 2, D, 11 + li)[1][grp]
                        fr = np.array([lay.filterRegions[r] for r in grp], np.int32)
                        tr = np.array([lay.sharedRegions[r] for r in grp], np.int32)
                        P = E.make_plan(fr, tr)
                        img = np.full((H, W), -1.0, np.float32)
                        P.eval_host(planes, img, with_check=True)
                        offs = np.concatenate([[0], np.cumsum(tr[:, 2].astype(np.int64) * tr[:, 3])])
                        d_tiles = devmem.zeros((int(offs[-1]),), -1.0)
                        P.eval_device_tiles(planes, devmem.ptr(d_tiles), with_check=True)
                        E.sync()
                        tiles = np.asarray(devmem.download(d_tiles), np.float32)
                        del d_tiles
                        P.close()
                        big = int(np.argmax(fr[:, 2].astype(np.int64) * fr[:, 3]))
                        far = int(np.argmax((tr[:, 0] + tr[:, 2]) * 100000 + tr[:, 1] + tr[:, 3]))
                        pick = sorted({big, far} | set(int(i) for i in rng.choice(len(grp), size=min(len(grp), 2), replace=False)))
                        fk = C.FILTER_BILATERAL if filt == "BL" else C.FILTER_NONE
                        q, s = C.filter_unary_batch(0, fr[pick], tr[pick], planes[pick], with_check=True, filter=fk, windR=windR, sig2=SIG2)
                        for i in pick:
                            x, y, w, h = tr[i]
                            got = img[y:y + h, x:x + w]
                            assert np.array_equal(bits(got.ravel()), bits(tiles[offs[i]:offs[i + 1]])), \
                                f"{filt!r} layer {li} cell {grp[i]}: device tiles differ from the host image output"
                            worst = max(worst, FC.compare(got, q[y:y + h, x:x + w], s[y:y + h, x:x + w], filt == "",
                                                          f"{filt!r} layer {li} group {gi} cell {grp[i]}"))
                            n_cells, n_px = n_cells + 1, n_px + int(w * h)
                            if (x + w, y + h) == (W, H):
                                corner_layers.add(li)
            finally:
                E.close()
            assert corner_layers == {0, 1, 2}, "a cell reaching the bottom-right corner in every layer"
            print(f"{filt!r} 2048 x 1536 x 256: {n_cells} cells, {n_px} pixels, worst |d| / sum w|p| {worst:.2e}")
    finally:
        C.close()
    print(f"  {time.perf_counter() - t0:.1f} s in all")


def test_warm_start_at_the_benchmark_size(bench_scene):
    """lexp_pm_init_from_labeling with "BL" on a random plane per pixel of the whole image: ~2000 seeded pixels against the oracle
    and bit for bit against the unary call (F(p), {p})."""
    import filter_checks as FC
    imL, vol, vol_host, windR = bench_scene
    D, (H, W) = int(vol.shape[0]), imL.shape[:2]
    t0 = time.perf_counter()
    worst = FC.check_warm_start("cv", "bl", H, W, D, windR, unary_pixels=2000, scene=(imL, None, vol_host, None))
    print(f"warm start 'BL' 2048 x 1536 x 256: worst |d| / sum w|p| {worst:.2e}; {time.perf_counter() - t0:.1f} s")


# ---- the right view at scale, the image-based energy at the demo geometry -----------------------------------------------------------------
def test_every_step_of_the_right_view_at_scale(devmem):
    """960 x 544 x 96, windR 32 (the scene of test_every_step_of_the_r16_instantiation), mode 1, "BL", two iterations: the second
    starts from a state the first has moved, and its Expansion proposals read planes the first wrote.  The initialisation and the
    steps of layer 2 certified (the FP64 bilateral oracle of a step sums ~10^9 weighted terms on the host), the other steps issued
    one by one, the final state against the twin's."""
    from localexpstereo_b200.sweep import V3_PROPOSERS_DEVICE
    scene_filter_sweep(devmem, "cv", "BL", 1, 544, 960, 96, 32, None, V3_PROPOSERS_DEVICE, iterations=2, seed=5, layers=(2,))


@pytest.mark.parametrize("mode", [0, 1])
def test_every_step_of_the_cones_pair_with_paramsBF(devmem, mode):
    """The initialisation and layer 25 certified, layers 5 and 15 issued one by one uncertified, the final state against the twin's."""
    scene_cones_bf(devmem, mode, layers=(2,))
