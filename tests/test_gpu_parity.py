"""GPU parity: CUDA path (through the C-ABI) vs the numpy oracle on identical seeded inputs."""
import numpy as np
import pytest

from oracle import lexp_oracle as O
from lexp_testlib import TorchDeviceMemory, assert_costs_close, make_scene, random_planes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scene():
    import localexpstereo_b200 as L
    H, W, D, windR = 150, 210, 24, 20
    imL, imR, volL, volR = make_scene(H, W, D)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.CostVolumeEnergy(imL, imR, volL, volR, prm, D - 1)
    Or = O.CostVolumeEnergyOracle(imL, imR, volL, volR, windR, 1e-4, 0.5, D - 1)
    yield dict(H=H, W=W, D=D, windR=windR, E=E, O=Or, L=L)
    E.close()


def test_stats_match_oracle(scene):
    for mode in (0, 1):
        got = scene["E"].stats(mode)
        ref = scene["O"].filter[mode].stats_f32()
        assert np.abs(got[:3] - ref[:3]).max() < 2e-7            # window means in [0, 1]
        scale = np.abs(ref[3:]).max(axis=0, keepdims=True)       # per-pixel norm of the inverse covariance
        assert (np.abs(got[3:] - ref[3:]) / scale).max() < 1e-6


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("unit", [10, 31])
def test_cells_of_a_layer(scene, mode, unit):
    L, E, Or = scene["L"], scene["E"], scene["O"]
    lm = L.LayerManager(scene["W"], scene["H"], scene["windR"])
    lay = lm.addLayer(unit)
    rng = O.CvRNG(7 + unit + mode)
    worst = 0.0
    for g in lay.disjointRegionSets[:6]:
        planes = random_planes(rng, [lay.unitRegions[r] for r in g], scene["D"])
        fr = [lay.filterRegions[r] for r in g]
        tr = [lay.sharedRegions[r] for r in g]
        img = np.full((scene["H"], scene["W"]), -7.0, np.float32)
        E.ComputeUnaryPotentialBatch(fr, tr, img, planes, mode=mode, with_check=True)
        touched = np.zeros_like(img, dtype=bool)
        for f, t, p in zip(fr, tr, planes):
            ref = Or.compute_unary_potential(f, t, p, mode)
            got = img[t[1]:t[1] + t[3], t[0]:t[0] + t[2]]
            worst = max(worst, assert_costs_close(got, ref, f"cell f={f} t={t}"))
            touched[t[1]:t[1] + t[3], t[0]:t[0] + t[2]] = True
        assert (img[~touched] == -7.0).all(), "wrote outside targetRect"
    print("worst rel err", worst)


def test_single_cell_virtuals(scene):
    """The two StereoEnergy virtuals, called the way FastGCStereo.h:49 / :113 does."""
    L, E, Or = scene["L"], scene["E"], scene["O"]
    H, W, D = scene["H"], scene["W"], scene["D"]
    rng = O.CvRNG(99)
    proposal = np.zeros((H, W), np.float32)
    for (f, t) in [((30, 20, 100, 90), (50, 40, 60, 50)), ((0, 0, 70, 60), (0, 0, 50, 40)), ((110, 60, 100, 90), (130, 80, 80, 70)),
                   ((40, 40, 41, 41), (60, 60, 1, 1))]:
        p = O.create_random_label(rng, t[0], t[1], 0, D - 1)
        view = proposal[f[1]:f[1] + f[3], f[0]:f[0] + f[2]]
        E.ComputeUnaryPotentialWithoutCheck(f, t, view, p)
        ref = Or.compute_unary_potential_without_check(f, t, p)
        assert_costs_close(proposal[t[1]:t[1] + t[3], t[0]:t[0] + t[2]], ref, f"nocheck {f} {t}")
        E.ComputeUnaryPotential(f, t, view, p)
        ref = Or.compute_unary_potential(f, t, p)
        assert_costs_close(proposal[t[1]:t[1] + t[3], t[0]:t[0] + t[2]], ref, f"check {f} {t}")


def test_branches_of_the_sampler(scene):
    """d < MIN, d >= MAX, NaN planes, invalid-corner mask (CostVolumeEnergy.h:78-92, StereoEnergy.h:577-610)."""
    E, Or, D = scene["E"], scene["O"], scene["D"]
    f, t = (20, 10, 120, 100), (40, 30, 80, 60)
    H, W = scene["H"], scene["W"]
    planes = [
        (0.0, 0.0, -5.0, 0.0),            # everywhere below MIN
        (0.0, 0.0, D + 3.0, 0.0),         # everywhere above MAX
        (0.35, -0.2, 3.0, 0.0),           # crosses both ends
        (float("nan"), 0.0, 1.0, 0.0),    # NaN disparity
        (0.0, 0.0, float(D - 1), 0.0),    # exactly MAX
        (0.0, 0.0, 0.0, 0.0),             # exactly MIN
        (1.7, 1.7, -100.0, 0.0),          # steep
        (0.0, 0.0, 5.5, float("inf")),    # v = inf poisons channelSum
    ]
    for p in planes:
        p = np.array(p, np.float32)
        for chk in (False, True):
            img = np.zeros((H, W), np.float32)
            view = img[f[1]:f[1] + f[3], f[0]:f[0] + f[2]]
            (E.ComputeUnaryPotential if chk else E.ComputeUnaryPotentialWithoutCheck)(f, t, view, p)
            ref = (Or.compute_unary_potential if chk else Or.compute_unary_potential_without_check)(f, t, p)
            got = img[t[1]:t[1] + t[3], t[0]:t[0] + t[2]]
            if np.isnan(ref).any():
                assert np.array_equal(np.isnan(ref), np.isnan(got))
                ref = np.nan_to_num(ref, nan=0.0); got = np.nan_to_num(got, nan=0.0)
            assert_costs_close(got, ref, f"plane {p} chk={chk}")


def test_filter_rect_smaller_than_dependency_cone(scene):
    """N is clipped at the *filterRect* (GuidedFilter.h:324), also when filterRect < targetRect +- 2R."""
    E, Or, D = scene["E"], scene["O"], scene["D"]
    H, W = scene["H"], scene["W"]
    rng = O.CvRNG(3)
    for (f, t) in [((50, 40, 60, 50), (55, 45, 50, 40)), ((50, 40, 60, 50), (50, 40, 60, 50)), ((10, 10, 25, 130), (12, 30, 20, 90))]:
        p = O.create_random_label(rng, t[0], t[1], 0, D - 1)
        img = np.zeros((H, W), np.float32)
        E.ComputeUnaryPotential(f, t, img[f[1]:f[1] + f[3], f[0]:f[0] + f[2]], p)
        ref = Or.compute_unary_potential(f, t, p)
        assert_costs_close(img[t[1]:t[1] + t[3], t[0]:t[0] + t[2]], ref, f"{f} {t}")


def test_errors_are_reported(scene):
    L, E = scene["L"], scene["E"]
    img = np.zeros((scene["H"], scene["W"]), np.float32)
    with pytest.raises(L.LexpError):
        E.ComputeUnaryPotentialBatch([(0, 0, 50, 50)], [(40, 40, 20, 20)], img, np.zeros((1, 4), np.float32))  # target not inside filter
    with pytest.raises(L.LexpError):
        E.ComputeUnaryPotentialBatch([(-5, 0, 50, 50)], [(0, 0, 20, 20)], img, np.zeros((1, 4), np.float32))  # outside the image


def test_concurrent_single_cell_calls_like_the_openmp_loop(scene):
    """FastGCStereo.h:30-49: N host threads call the virtual concurrently, one cell each, K proposals per cell, all writing
    disjoint targetRects of one proposalCost image.  Must equal the batched evaluation (and exercises the per-cell plan cache)."""
    from concurrent.futures import ThreadPoolExecutor
    L, E = scene["L"], scene["E"]
    H, W, D = scene["H"], scene["W"], scene["D"]
    lay = L.LayerManager(W, H, scene["windR"]).addLayer(12)
    g = lay.disjointRegionSets[2]
    rng = O.CvRNG(41)
    for step in range(3):
        planes = random_planes(rng, [lay.unitRegions[r] for r in g], D)
        ref = np.zeros((H, W), np.float32)
        E.ComputeUnaryPotentialBatch([lay.filterRegions[r] for r in g], [lay.sharedRegions[r] for r in g], ref, planes)
        img = np.zeros((H, W), np.float32)

        def one(i):
            f, t = lay.filterRegions[g[i]], lay.sharedRegions[g[i]]
            E.ComputeUnaryPotential(f, t, img[f[1]:f[1] + f[3], f[0]:f[0] + f[2]], planes[i])

        with ThreadPoolExecutor(max_workers=8) as ex:
            list(ex.map(one, range(len(g))))
        assert np.array_equal(img, ref)


@pytest.mark.parametrize("windR", [8, 13, 32])
def test_other_filter_radii(windR):
    """R = windR / 2 = 4 and 6 run the generic (runtime-R) kernel, R = 16 the second specialised one (config 5: windR 32)."""
    import localexpstereo_b200 as L
    H, W, D = 140, 190, 20
    imL, imR, volL, volR = make_scene(H, W, D, seed=windR)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.CostVolumeEnergy(imL, imR, volL, volR, prm, D - 1)
    Or = O.CostVolumeEnergyOracle(imL, imR, volL, volR, windR, 1e-4, 0.5, D - 1)
    lay = L.LayerManager(W, H, windR).addLayer(23)
    rng = O.CvRNG(windR)
    worst = 0.0
    for mode, g in ((0, lay.disjointRegionSets[0]), (1, lay.disjointRegionSets[5]), (0, lay.disjointRegionSets[-1])):
        planes = random_planes(rng, [lay.unitRegions[r] for r in g], D)
        fr = [lay.filterRegions[r] for r in g]
        tr = [lay.sharedRegions[r] for r in g]
        img = np.zeros((H, W), np.float32)
        E.ComputeUnaryPotentialBatch(fr, tr, img, planes, mode=mode)
        for f, t, p in zip(fr, tr, planes):
            worst = max(worst, assert_costs_close(img[t[1]:t[1] + t[3], t[0]:t[0] + t[2]], Or.compute_unary_potential(f, t, p, mode), f"windR {windR} {f}"))
    print("windR", windR, "worst rel err", worst)
    E.close()


def test_nonzero_min_disparity_and_odd_max(scene):
    """MIN_DISPARITY != 0 / MAX_DISPARITY != D-1 take the generic sampler (D0 offset, CostVolumeEnergy.h:67,83)."""
    import localexpstereo_b200 as L
    H, W, D = 100, 130, 16
    imL, imR, volL, volR = make_scene(H, W, D, seed=77)
    prm = L.Parameters(windR=20, filterName="GF", filter_param1=1e-4, th_col=0.6)
    for (mn, mx) in [(-4.0, 11.0), (0.0, 9.0)]:
        E = L.CostVolumeEnergy(imL, imR, volL, volR, prm, mx, mn)
        Or = O.CostVolumeEnergyOracle(imL, imR, volL, volR, 20, 1e-4, 0.6, mx, mn)
        f, t = (10, 5, 110, 90), (30, 25, 70, 50)
        for p in [(0.05, 0.02, 1.0, 0), (0.0, 0.0, -2.5, 0), (0.2, -0.1, 4.0, 0), (0.0, 0.0, 10.5, 0)]:
            p = np.array(p, np.float32)
            img = np.zeros((H, W), np.float32)
            E.ComputeUnaryPotential(f, t, img[f[1]:f[1] + f[3], f[0]:f[0] + f[2]], p)
            ref = Or.compute_unary_potential(f, t, p)
            assert_costs_close(img[t[1]:t[1] + t[3], t[0]:t[0] + t[2]], ref, f"min {mn} max {mx} plane {p}")
        E.close()


@pytest.fixture(scope="module")
def devmem():
    return TorchDeviceMemory()


def test_device_image_and_tile_outputs(scene, devmem):
    """lexp_plan_eval_device (H x W cost image in device memory, host or device planes) and lexp_plan_eval_device_tiles
    (per-call contiguous tiles = the all-gather payload of the cell shard, sweep.tile_offsets) against the host path."""
    from localexpstereo_b200.sweep import tile_offsets
    L, E = scene["L"], scene["E"]
    H, W, D = scene["H"], scene["W"], scene["D"]
    lay = L.LayerManager(W, H, scene["windR"]).addLayer(14)
    g = lay.disjointRegionSets[1]
    fr = [lay.filterRegions[r] for r in g]
    tr = [lay.sharedRegions[r] for r in g]
    plan = E.make_plan(fr, tr)
    rng = O.CvRNG(77)
    offs, total = tile_offsets(tr)
    for mode in (0, 1):
        planes = random_planes(rng, [lay.unitRegions[r] for r in g], D)
        ref = np.full((H, W), -7.0, np.float32)
        plan.eval_host(planes, ref, True, mode)
        # device image, host planes; padded pitch
        pitch = (W + 13) * 4
        d_img = devmem.zeros((H, W + 13), -7.0)
        plan.eval_device(planes, devmem.ptr(d_img), pitch, True, mode)
        E.sync()
        got = devmem.download(d_img)
        assert np.array_equal(got[:, :W], ref) and (got[:, W:] == -7.0).all()
        # device image, device planes
        d_pl = devmem.upload(np.asarray(planes, np.float32))
        d_img2 = devmem.zeros((H, W), -7.0)
        plan.eval_device(devmem.ptr(d_pl), devmem.ptr(d_img2), W * 4, True, mode, planes_on_device=True)
        E.sync()
        assert np.array_equal(devmem.download(d_img2), ref)
        # tiles
        d_tiles = devmem.zeros((total + 5,), -9.0)
        plan.eval_device_tiles(planes, devmem.ptr(d_tiles), True, mode)
        E.sync()
        tiles = devmem.download(d_tiles)
        assert (tiles[total:] == -9.0).all()
        for (x, y, w, h), o in zip(tr, offs):
            assert np.array_equal(tiles[o:o + w * h].reshape(h, w), ref[y:y + h, x:x + w])
    plan.close()


def test_host_tile_output(scene):
    """lexp_plan_eval_host_tiles: per-call contiguous tiles in host memory, zero-copy (registered buffer) and staged, against
    the H x W image path; a cv::Mat-style header over tile i is what the restructured fusion loop reads (INTEGRATION.md 3)."""
    from localexpstereo_b200.sweep import tile_offsets
    L, E = scene["L"], scene["E"]
    H, W, D = scene["H"], scene["W"], scene["D"]
    lay = L.LayerManager(W, H, scene["windR"]).addLayer(11)
    g = lay.disjointRegionSets[3]
    fr = [lay.filterRegions[r] for r in g]
    tr = [lay.sharedRegions[r] for r in g]
    plan = E.make_plan(fr, tr)
    offs, total = tile_offsets(tr)
    assert total == plan.target_px
    rng = O.CvRNG(55)
    for mode in (0, 1):
        planes = random_planes(rng, [lay.unitRegions[r] for r in g], D)
        ref = np.full((H, W), -7.0, np.float32)
        plan.eval_host(planes, ref, True, mode)
        staged = np.full(total + 3, -9.0, np.float32)
        plan.eval_host_tiles(planes, staged, True, mode)
        mapped = np.full(total + 3, -9.0, np.float32)
        L.host_register(mapped)
        try:
            plan.eval_host_tiles(planes, mapped, True, mode)
        finally:
            L.host_unregister(mapped)
        assert np.array_equal(staged, mapped) and (staged[total:] == -9.0).all()
        for (x, y, w, h), o in zip(tr, offs):
            assert np.array_equal(staged[o:o + w * h].reshape(h, w), ref[y:y + h, x:x + w])
    plan.close()


def test_partially_registered_output_takes_the_staged_path(scene):
    """Only the FIRST part of the cost image / tile buffer is page-locked (it starts inside somebody's registration): the zero-copy
    path must not be taken -- a kernel writing through that alias would run past the end of the mapping (an illegal address on the
    device) -- and the staged path must deliver the same pixels."""
    from localexpstereo_b200.sweep import tile_offsets
    L, E = scene["L"], scene["E"]
    H, W, D = scene["H"], scene["W"], scene["D"]
    lay = L.LayerManager(W, H, scene["windR"]).addLayer(11)
    g = lay.disjointRegionSets[1]
    fr = [lay.filterRegions[r] for r in g]
    tr = [lay.sharedRegions[r] for r in g]
    plan = E.make_plan(fr, tr)
    rng = O.CvRNG(56)
    planes = random_planes(rng, [lay.unitRegions[r] for r in g], D)
    ref = np.full((H, W), -7.0, np.float32)
    plan.eval_host(planes, ref, True, 0)
    part = np.full((H, W), -7.0, np.float32)
    head = part[:max(1, min(t[1] for t in tr) + 2)]          # the image's first rows only: the range the calls write is longer
    L.host_register(head)
    try:
        plan.eval_host(planes, part, True, 0)
    finally:
        L.host_unregister(head)
    assert np.array_equal(part, ref)
    _, total = tile_offsets(tr)
    tiles_ref = np.full(total, -9.0, np.float32)
    plan.eval_host_tiles(planes, tiles_ref, True, 0)
    tiles = np.full(total, -9.0, np.float32)
    L.host_register(tiles[:total // 2])
    try:
        plan.eval_host_tiles(planes, tiles, True, 0)
    finally:
        L.host_unregister(tiles[:total // 2])
    assert np.array_equal(tiles, tiles_ref)
    plan.close()


def _textureless_guides(H, W):
    """Guides on which the 3x3 covariance is (nearly) singular: the FP32 hazard SURVEY.md section 7 names."""
    const = np.full((H, W, 3), 128, np.uint8)
    two = np.full((H, W, 3), 40, np.uint8); two[:, W // 2:] = 200                      # one vertical step edge
    ramp = np.zeros((H, W, 3), np.uint8); ramp[:] = (np.arange(W) * 255 // (W - 1)).astype(np.uint8)[None, :, None]
    sat = np.full((H, W, 3), 255, np.uint8); sat[H // 3:2 * H // 3, W // 4:W // 2] = 0  # saturated black / white blocks
    chan = np.zeros((H, W, 3), np.uint8); chan[..., 0] = 255; chan[::2, :, 1] = 7       # one constant channel, one 2-level
    return {"constant": const, "two_level": two, "ramp": ramp, "saturated": sat, "channel": chan}


@pytest.mark.parametrize("name", ["constant", "two_level", "ramp", "saturated", "channel"])
def test_textureless_guides(name):
    """Constant / two-level / saturated guide images: the covariance is eps*I (or rank 1 + eps*I), inv-covariance entries
    reach 1/eps = 1e4 and the (a, b) coefficients are differences of nearly equal numbers -- FP32 filter vs the FP64 oracle."""
    import localexpstereo_b200 as L
    H, W, D, windR = 120, 150, 16, 20
    g = _textureless_guides(H, W)[name]
    volL = O.synthetic_volume(D, H, W, 77)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.CostVolumeEnergy(g, None, volL, None, prm, D - 1)
    try:
        Or = O.CostVolumeEnergyOracle(g, None, volL, None, windR, 1e-4, 0.5, D - 1)
        rng = O.CvRNG(5)
        worst = 0.0
        for (f, t) in [((0, 0, 100, 90), (0, 0, 60, 50)), ((30, 20, 120, 100), (50, 40, 80, 60)), ((60, 40, 90, 80), (80, 60, 50, 40))]:
            for _ in range(3):
                p = O.create_random_label(rng, t[0] + 5, t[1] + 5, 0, D - 1)
                img = np.zeros((H, W), np.float32)
                E.ComputeUnaryPotential(f, t, img[f[1]:f[1] + f[3], f[0]:f[0] + f[2]], p)
                ref = Or.compute_unary_potential(f, t, p)
                worst = max(worst, assert_costs_close(img[t[1]:t[1] + t[3], t[0]:t[0] + t[2]], ref, f"{name} {f} {t}"))
        print(name, "worst rel err", worst)
    finally:
        E.close()


def test_plan_outlives_its_energy():
    """lexp_destroy orphans the plans that are still alive (ADVICE r1): closing the energy first must stay safe."""
    import localexpstereo_b200 as L
    H, W, D = 64, 80, 8
    imL, _, volL, _ = make_scene(H, W, D)
    E = L.CostVolumeEnergy(imL, None, volL, None, L.Parameters(windR=8, filterName="GF", filter_param1=1e-4, th_col=0.5), D - 1)
    plan = E.make_plan([(0, 0, 40, 40)], [(8, 8, 20, 20)])
    img = np.zeros((H, W), np.float32)
    plan.eval_host(np.array([[0, 0, 3.0, 0]], np.float32), img, True, 0)
    E.close()
    with pytest.raises(L.LexpError):
        plan.eval_host(np.array([[0, 0, 3.0, 0]], np.float32), img, True, 0)   # the context is gone: an error, not a crash
    plan.close()


def test_volume_preparation_on_the_device(devmem):
    """SURVEY.md 8 f-4: fillOutOfView / convertVolumeL2R (main.cpp:146-199) fused into the upload's re-layout pass.  The energy
    built from the raw left volume with LEXP_VOL_FILL (view 0) and LEXP_VOL_RIGHT_FROM_LEFT (view 1) must produce exactly the costs
    of an energy that was given the volumes prepared on the host by the oracle's restatement of the two functions; host upload in
    several slabs (LEXP_UPLOAD_SLAB_MB) and the device-pointer path."""
    import os
    import localexpstereo_b200 as L
    H, W, D, windR = 70, 95, 21, 12     # W not a multiple of 4, D not a multiple of 8: ragged blocks and slabs
    imL, imR, volL, _ = make_scene(H, W, D)
    prepL = O.fill_out_of_view(volL.copy(), 0)
    prepR = O.fill_out_of_view(O.convert_volume_l2r(prepL), 1)
    assert np.array_equal(prepR, np.stack([volL[d][:, np.minimum(np.arange(W) + d, W - 1)] for d in range(D)]))   # the closed form the kernel uses
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    ref = L.CostVolumeEnergy(imL, imR, prepL, prepR, prm, D - 1)
    old = os.environ.get("LEXP_UPLOAD_SLAB_MB")
    os.environ["LEXP_UPLOAD_SLAB_MB"] = "0"     # smallest slab (8 disparities): 3 slabs, the last one ragged
    try:
        got = L.CostVolumeEnergy(imL, imR, None, None, prm, D - 1)
        got.set_volume(0, volL, L.VOL_FILL)
        got.set_volume(1, volL, L.VOL_RIGHT_FROM_LEFT)
        dev = L.CostVolumeEnergy(imL, imR, None, None, prm, D - 1)
        d_vol = devmem.upload(volL)
        dev.set_volume(0, d_vol if hasattr(d_vol, "is_cuda") else volL, L.VOL_FILL)
        dev.set_volume(1, d_vol if hasattr(d_vol, "is_cuda") else volL, L.VOL_RIGHT_FROM_LEFT)
    finally:
        if old is None:
            os.environ.pop("LEXP_UPLOAD_SLAB_MB")
        else:
            os.environ["LEXP_UPLOAD_SLAB_MB"] = old
    try:
        lay = L.LayerManager(W, H, windR).addLayer(9)
        rng = O.CvRNG(4)
        for mode in (0, 1):
            g = lay.disjointRegionSets[3 + mode]
            planes = random_planes(rng, [lay.unitRegions[r] for r in g], D)
            fr, tr = [lay.filterRegions[r] for r in g], [lay.sharedRegions[r] for r in g]
            imgs = []
            for E in (ref, got, dev):
                img = np.full((H, W), -7.0, np.float32)
                E.ComputeUnaryPotentialBatch(fr, tr, img, planes, mode=mode)
                imgs.append(img)
            assert np.array_equal(imgs[0], imgs[1]) and np.array_equal(imgs[0], imgs[2]) and (imgs[0] != -7.0).any()
        with pytest.raises(L.LexpError):
            got.set_volume(0, volL, L.VOL_RIGHT_FROM_LEFT)   # the derived volume is view 1's
    finally:
        for E in (ref, got, dev):
            E.close()


def test_volume_file_disparity_map_and_pfm(tmp_path):
    """SURVEY.md 8 f-4, the formats either side of the path: the reference's cost-volume file (`im0.acrt`: raw float[D][H][W],
    main.cpp:353-364) streamed from disk in several slabs with the volume preparation fused in must give exactly the costs of the
    same array uploaded from memory; computeDisparities of the device state (StereoEnergy.h:269-272) and the PFM file the
    reference writes from it (main.cpp:319,410; Utilities.hpp:84-137: header "Pf / w h / -1/255", rows bottom-up)."""
    import os
    import localexpstereo_b200 as L
    H, W, D, windR = 66, 91, 19, 12
    imL, imR, volL, _ = make_scene(H, W, D, seed=12)
    path = os.path.join(str(tmp_path), "im0.acrt")
    volL.tofile(path)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    old = os.environ.get("LEXP_UPLOAD_SLAB_MB")
    os.environ["LEXP_UPLOAD_SLAB_MB"] = "0"      # 8 disparities per slab: three slabs, the last one ragged
    A = L.CostVolumeEnergy(imL, imR, None, None, prm, D - 1)
    B = L.CostVolumeEnergy(imL, imR, None, None, prm, D - 1)
    try:
        A.set_volume(0, volL, L.VOL_FILL); A.set_volume(1, volL, L.VOL_RIGHT_FROM_LEFT)
        B.set_volume_file(0, path, L.VOL_FILL); B.set_volume_file(1, path, L.VOL_RIGHT_FROM_LEFT)
    finally:
        if old is None:
            os.environ.pop("LEXP_UPLOAD_SLAB_MB")
        else:
            os.environ["LEXP_UPLOAD_SLAB_MB"] = old
    try:
        lay = L.LayerManager(W, H, windR).addLayer(9)
        rng = O.CvRNG(2)
        for mode in (0, 1):
            g = lay.disjointRegionSets[2 + mode]
            planes = random_planes(rng, [lay.unitRegions[r] for r in g], D)
            fr, tr = [lay.filterRegions[r] for r in g], [lay.sharedRegions[r] for r in g]
            ia, ib = np.full((H, W), -7.0, np.float32), np.full((H, W), -7.0, np.float32)
            A.ComputeUnaryPotentialBatch(fr, tr, ia, planes, mode=mode)
            B.ComputeUnaryPotentialBatch(fr, tr, ib, planes, mode=mode)
            assert np.array_equal(ia, ib) and (ia != -7.0).any()
        with open(os.path.join(str(tmp_path), "short.acrt"), "wb") as f:
            f.write(volL.tobytes()[:-4])
        with pytest.raises(L.LexpError):
            B.set_volume_file(0, os.path.join(str(tmp_path), "short.acrt"))          # not float[D][H][W] of this size
        with pytest.raises(L.LexpError):
            B.set_volume_file(0, os.path.join(str(tmp_path), "absent.acrt"))
        # disparity map of a labeling + the PFM file
        lab = np.zeros((H, W, 4), np.float32)
        for y in range(0, H, 5):
            for x in range(0, W, 7):
                lab[y:y + 5, x:x + 7] = O.create_random_label(rng, x, y, 0.0, D - 1.0)
        B.pm_begin(0, np.zeros((H, W), np.float32), lab)
        disp = B.computeDisparities(0)
        xs, ys = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32))
        want = ((xs * lab[..., 0] + ys * lab[..., 1]) + lab[..., 2]) + np.float32(0) * lab[..., 3]   # channelDot(coordinates, labeling)
        assert np.array_equal(disp, want)
        pfm = os.path.join(str(tmp_path), "disp0.pfm")
        L.save_pfm_file(pfm, disp)
        raw = open(pfm, "rb").read()
        head = ("Pf\n%d %d\n%f\n" % (W, H, -1.0 / 255.0)).encode()
        assert raw.startswith(head) and len(raw) == len(head) + H * W * 4
        assert np.array_equal(np.frombuffer(raw[len(head):], np.float32).reshape(H, W)[::-1], disp)
    finally:
        A.close(); B.close()
