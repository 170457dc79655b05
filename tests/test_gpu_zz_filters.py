"""The bilateral filter ("BL" / "BF") and the unfiltered mode ("") on the H100 (lexp_filters.cuh, DESIGN.md 3i): the unary calls
through every output path, the warm start and the PatchMatch steps of both energies against the FP64 oracle (tests/filter_checks.py),
sampled cells of large images, CUDA-graph replay, concurrent lexp_eval_cell calls, and whole runs against the same runs issued through
the public calls (tests/run_checks.py)."""
import threading

import numpy as np
import pytest

import localexpstereo_b200 as L
import filter_checks as FC
import run_checks as RC
from lexp_testlib import TorchDeviceMemory, bits, make_scene

pytestmark = pytest.mark.gpu
KINDS = [("cv", "bl"), ("cv", "none"), ("naive", "bl"), ("naive", "none")]


@pytest.fixture(scope="module")
def devmem():
    return TorchDeviceMemory()


@pytest.mark.parametrize("energy,filt", KINDS)
@pytest.mark.parametrize("mode", [0, 1])
def test_unary_calls(devmem, energy, filt, mode):
    FC.check_unary(devmem, energy, filt, 61, 83, 16, 20, mode=mode, seed=mode)


@pytest.mark.parametrize("windR", [2, 5, 21, 49])
def test_unary_radii(devmem, windR):
    FC.check_unary(devmem, "cv", "bl", 70, 120, 12, windR, seed=windR)
    FC.check_unary(devmem, "naive", "bl", 70, 120, 12, windR, seed=windR)


def test_unary_min_disparity(devmem):
    FC.check_unary(devmem, "cv", "none", 40, 64, 24, 5, MIN=3.0, MAX=17.5)
    FC.check_unary(devmem, "cv", "bl", 40, 64, 24, 5, MIN=3.0, MAX=17.5)


@pytest.mark.parametrize("energy,filt", KINDS)
def test_warm_start(energy, filt):
    FC.check_warm_start(energy, filt, 41, 57, 12, 6, mode=1 if energy == "naive" else 0)


@pytest.mark.parametrize("energy,filt", KINDS)
def test_pm_steps(devmem, energy, filt):
    FC.check_pm_steps(devmem, energy, filt, 80, 104, 24, 6, unit=10)


@pytest.mark.parametrize("H,W,D,windR,unit", [(544, 960, 96, 32, 25), (991, 1437, 64, 20, 25)])
def test_large_layer_sampled(devmem, H, W, D, windR, unit):
    """A whole group of layer-0 cells of a large image on the device; the largest filterRect and a border cell against the oracle
    on sampled pixels of their targetRects, both filters of the cost-volume energy."""
    scene = make_scene(H, W, D, seed=3)
    for filt in ("bl", "none"):
        E, Or = FC.make("cv", filt, H, W, D, windR, scene=scene)
        try:
            ly = L.LayerManager(W, H, windR).addLayer(unit)
            cells = ly.disjointRegionSets[0]
            fr = np.array([ly.filterRegions[i] for i in cells], np.int32)
            tr = np.array([ly.sharedRegions[i] for i in cells], np.int32)
            rng = np.random.default_rng(5)
            planes = FC.plan_planes(len(cells), H, W, 0.0, D - 1.0, 9)
            planes[3:5] = planes[0]                  # plan_planes puts NaN / inf there: keep the sampled cells' planes finite
            P = E.make_plan(fr, tr)
            img = np.full((H, W), -1.0, np.float32)
            P.eval_host(planes, img, with_check=True)
            big = int(np.argmax(fr[:, 2] * fr[:, 3]))
            for i in {0, big}:
                x, y, w, h = tr[i]
                for _ in range(6):
                    px, py = int(x + rng.integers(w)), int(y + rng.integers(h))
                    q, s = Or.unary(tuple(fr[i]), (px, py, 1, 1), planes[i])
                    FC.compare(img[py:py + 1, px:px + 1], q, s, filt == "none", f"{H}x{W} cell {i} ({px},{py})")
            P.close()
        finally:
            E.close()


@pytest.mark.parametrize("energy,filt", [("cv", "bl"), ("naive", "bl")])
def test_graph_replay_and_concurrent_cells(devmem, energy, filt):
    """A CUDA graph of a plan evaluation replays the direct launch bit for bit; concurrent lexp_eval_cell calls from several threads
    (combined into batched launches) give each call's direct result."""
    import torch
    H, W, D, windR = 64, 96, 16, 8
    E, _ = FC.make(energy, filt, H, W, D, windR)
    try:
        fr, tr = FC.corner_calls(H, W, windR)
        planes = FC.plan_planes(len(fr), H, W, 0.0, D - 1.0, 11, v=energy == "naive")
        P = E.make_plan(fr, tr)
        ref = np.full((H, W), -1.0, np.float32)
        P.eval_host(planes, ref)
        d_pl = devmem.upload(planes)
        out = devmem.zeros((H, W), -1.0)
        s = torch.cuda.Stream()
        E.set_stream(s.cuda_stream)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            P.eval_device(devmem.ptr(d_pl), devmem.ptr(out), W * 4, planes_on_device=True)
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(bits(devmem.download(out)), bits(ref))
        res = [None] * len(fr)

        def one(i):
            f, t = fr[i], tr[i]
            c = np.full((f[3], f[2]), -1.0, np.float32)
            E.ComputeUnaryPotential(tuple(f), tuple(t), c, planes[i])
            res[i] = c[t[1] - f[1]:t[1] - f[1] + t[3], t[0] - f[0]:t[0] - f[0] + t[2]].copy()
        for _ in range(3):
            th = [threading.Thread(target=one, args=(i,)) for i in range(len(fr))]
            [t.start() for t in th]
            [t.join() for t in th]
            for i, (x, y, w, h) in enumerate(tr):
                assert np.array_equal(bits(res[i]), bits(ref[y:y + h, x:x + w])), i
        P.close()
    finally:
        E.close()


@pytest.mark.parametrize("energy,filt", KINDS)
def test_errors(energy, filt):
    FC.check_errors(energy, filt)


def _mk(naive, name, H=72, W=96, D=16, windR=5):
    def mk():
        imL, imR, volL, volR = make_scene(H, W, D)
        prm = L.Parameters(windR=windR, filterName=name, filter_param1=10.0, th_col=0.5)
        E = L.NaiveStereoEnergy(imL, imR, prm, D - 1) if naive else L.CostVolumeEnergy(imL, imR, volL, volR, prm, D - 1)
        E.set_smoothness(**RC.SMOOTH)
        return E
    return mk


@pytest.mark.parametrize("naive,name", [(False, "BL"), (False, ""), (True, "BF")])
@pytest.mark.parametrize("views", [(0,), (0, 1)])
def test_run_equals_composition(naive, name, views):
    """lexp_run bit for bit against its public calls; the energy never rises from one graph-cut iteration to the next."""
    lab, raw, calls = RC.check_run_equals_composition(_mk(naive, name), views, 1, 3, [5, 15], RC.PROPS, seed=11)
    for m in views:
        e = [r["energy"] for i, mm, r, _ in calls if mm == m and 1 <= i <= 4]
        assert all(b <= a * (1 + 1e-6) for a, b in zip(e, e[1:])), e


@pytest.mark.parametrize("energy,filt", KINDS)
def test_device_equals_the_compiled_reference(energy, filt):
    """The device's unary costs against the reference's own energy with this filterName (oracle/_ref/liblexp_ref_filters.so), on a
    designed scene at windR 5 and 20 and on the cones crop, both views."""
    from oracle import ref_filters
    if not ref_filters.available():
        pytest.skip("oracle/_ref/liblexp_ref_filters.so is not built")
    for mode in (0, 1):
        FC.check_against_reference(energy, filt, 47, 61, 10, 5, mode=mode, seed=mode, device=True)
        FC.check_against_reference(energy, filt, 60, 90, 12, 20, mode=mode, seed=2 + mode, device=True)
        FC.check_against_reference(energy, filt, 0, 0, 20, 10, mode=mode, scene=FC.cones_scene(), device=True)


def _gc_energy(naive, name):
    imL, imR, volL, volR = FC.cones_scene() if naive else make_scene(96, 128, 16, seed=4)
    D = 20 if naive else 16
    prm = L.Parameters(windR=8, filterName=name, filter_param1=10.0, th_col=0.5)
    return L.NaiveStereoEnergy(imL, imR, prm, D - 1) if naive else L.CostVolumeEnergy(imL, None, volL, None, prm, D - 1)


@pytest.mark.parametrize("naive,name", [(True, "BF"), (False, "BL"), (False, "")])
def test_every_graph_cut_move(devmem, naive, name):
    """One graph-cut iteration over two layers with the device proposers, every move certified (a)-(d) against the exact minimum cut
    of the same graph (lexp_replay.certify_gc_step, as tests/test_gpu_zz_gc_moves.py): the cones crop with the image-based energy and
    "BF", a synthetic cost-volume scene with "BL" and ""."""
    from localexpstereo_b200.sweep import GCSweep
    from lexp_replay import certify_gc_step
    from lexp_testlib import seeded_labels
    lam, th = 1.0, 1.0
    E = _gc_energy(naive, name)
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]]
    S = GCSweep(E, unit_sizes=[6, 18], proposers=props, lam=lam, omega=10.0, th_smooth=th, epsilon=0.01)
    try:
        S.begin()
        S.init(seeded_labels(S, 4))
        n_moves = 0
        for g in S.groups:
            for k, kind, m, sd in S.group_steps(g.layer, g.group, 0, 12):
                n_moves += len(certify_gc_step(E, g.plan, g.targets, 0, lam, th, devmem, kind=kind, m=m, seed=sd, ties_ok=True))
        assert n_moves > 100
    finally:
        S.close()
        E.close()


def test_cones_run_with_the_bilateral_filter():
    """-mode MiddV2 with paramsBF (Parameters(lambda, windR, "BF", 10)) on the MiddV2 cones pair: lexp_run equals the run composed from
    the public calls bit for bit; the energy never rises over the graph-cut iterations; the Evaluator's error rates are printed."""
    import os
    from localexpstereo_b200 import cli
    cones = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "middv2_cones")
    o = cli.parse_args(["-mode", "MiddV2", "-targetDir", cones])
    data = cli.load_data(cones + "/")
    imL, imR, gt, nonocc, ndisp, prec = data

    def mk():
        prm = L.Parameters(lambda_=o["smooth_weight"], windR=o["filterRadious"], filterName="BF", filter_param1=10.0)
        E = L.NaiveStereoEnergy(imL, imR, prm, float(ndisp - 1))
        E.set_smoothness(prm.lambda_, prm.omega, prm.th_smooth, prm.epsilon)
        return E
    from localexpstereo_b200.sweep import V3_PROPOSERS_REFERENCE
    lab, raw, calls = RC.check_run_equals_composition(mk, (0,), 1, 2, [5, 15, 25], V3_PROPOSERS_REFERENCE, seed=7)
    e = [r["energy"] for i, m, r, _ in calls if 1 <= i <= 3]
    assert all(b <= a * (1 + 1e-6) for a, b in zip(e, e[1:])), e
    E = mk()
    try:
        E.set_ground_truth(gt, nonocc)
        pts = []
        E.run(2, (0,), 1, None, [5, 15, 25], V3_PROPOSERS_REFERENCE, 7, prec, 0.5, callback=lambda i, m, r, t: pts.append((i, r)))
        for i, r in pts:
            print(f"cones BF point {i}: all {r['all']:.2f} %  nonocc {r['nonocc']:.2f} %  energy {r['energy']:.1f}")
    finally:
        E.close()
