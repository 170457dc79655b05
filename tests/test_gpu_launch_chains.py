"""The launch paths bench.py times, against fully serialized runs of the same work.

The benchmark issues its sweeps on the caller's stream, lets consecutive launches of lexp_fused_kernel overlap (programmatic
dependent launch: set_overlap for the unary sweep, always for the PatchMatch phase) and replays them from a CUDA graph.  Every test
here runs the same inputs, plans, planes and seeds a second time on a context created with LEXP_PDL_OFF=1, whose launches are
fully stream-serialised, and requires the results to be bit-identical.  CostVolumeEnergy.overlapped_launch_count proves that the
context under test really overlapped its launches (and the reference did not).

Scenes: the benchmark's default workload, the R = 16 instantiation (windR 32), a ragged generic-R case (W not a multiple of 4) and
the NaiveStereoEnergy workload (unary only).  tests/test_emu_launch_chains.py runs the tests without graphs or torch streams on
the emulator."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import lexp_oracle as O
from lexp_testlib import TorchDeviceMemory, assert_costs_close, pdl_off

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# name: W, H, D, windR; `units` / `steps`: the sweep's layers (default: sweep.v3_layer_units / V3_STEPS, as bench.py).
# bench_planes: the sweep's planes are bench.all_planes' exactly; otherwise their slopes are scaled by 0.1 about the unit centre
# (Scene.tempered): bench's steep planes leave a third of the pixels COST_FOR_INVALID in both of their last two writes at these
# disparity ranges, and a write that cannot be told from the one before it would hide a reordering.
SCENES = {
    "default_2048x1536x256_r20": dict(W=2048, H=1536, D=256, windR=20, device_volume=True, bench_planes=True),
    "r16_960x544x96_r32": dict(W=960, H=544, D=96, windR=32),
    "ragged_437x291x40_r12": dict(W=437, H=291, D=40, windR=12),
    "naive_450x375x64_r20": dict(W=450, H=375, D=64, windR=20, naive=True, units=[5, 15, 25]),
}
SMALL = ["ragged_437x291x40_r12", "naive_450x375x64_r20"]
PM_SCENES = [n for n, s in SCENES.items() if not s.get("naive")]
PM_SEED = 4321


class Scene:
    """Two contexts on the same inputs: E (overlapping launches allowed, on the caller's stream `stream` when given) and R
    (LEXP_PDL_OFF=1, its own stream); a UnarySweep of the benchmark's shape on each, and its planes on the device."""

    def __init__(self, devmem, stream, W, H, D, windR, naive=False, units=None, steps=None, device_volume=False, bench_planes=False):
        import localexpstereo_b200 as L
        from localexpstereo_b200 import synth
        from localexpstereo_b200.sweep import UnarySweep
        import bench
        self.W, self.H, self.D, self.windR, self.naive, self.devmem = W, H, D, windR, naive, devmem
        self.imL = synth.synthetic_image(H, W, 42)
        self.imR = synth.synthetic_image(H, W, 43) if naive else None
        self.vol = None
        if naive:
            prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4)
            make = lambda: L.NaiveStereoEnergy(self.imL, self.imR, prm, D - 1)   # noqa: E731
        else:
            if device_volume:   # as test_gpu_golden.full: generated on the device, complete before the contexts read it
                import torch
                g = torch.Generator(device="cuda").manual_seed(1234)
                vol = torch.rand((D, H, W), generator=g, device="cuda", dtype=torch.float32)
                torch.cuda.synchronize()
            else:
                vol = self.vol = np.random.default_rng(1234).random((D, H, W), dtype=np.float32)
            prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
            make = lambda: L.CostVolumeEnergy(self.imL, None, vol, None, prm, D - 1)   # noqa: E731
        self.E = make()
        with pdl_off():
            self.R = make()
        self.stream = stream
        if stream is not None:
            self.E.set_stream(stream.cuda_stream)   # before any capture: the context's own stream is released here
        self.E.set_overlap(True)                     # all plane arrays are on the device before the first launch (bench.py)
        self.units, self.steps = units, steps
        self.sweep = {id(E): UnarySweep(E, unit_sizes=units, steps=steps) for E in (self.E, self.R)}
        S = self.sweep[id(self.R)]
        self.planes_h = bench.all_planes(S, D) if bench_planes else self.tempered(bench.all_planes(S, D), S)
        self.planes_d = [devmem.upload(p) for p in self.planes_h]
        self.launches = S.launches_per_sweep
        self._ref = None

    @staticmethod
    def tempered(planes, S, scale=np.float32(0.1)):
        """planes [K][n][4] of every group with a and b scaled by `scale`, c moved so that the disparity at each unit's centre stays."""
        out = []
        for gi, g in enumerate(S.groups):
            u = np.array([S.layer(g.layer).unitRegions[r] for r in g.cells], np.float32)
            cx, cy = u[:, 0] + u[:, 2] * np.float32(0.5), u[:, 1] + u[:, 3] * np.float32(0.5)
            p = planes[gi].copy()
            z = p[..., 0] * cx + p[..., 1] * cy + p[..., 2]
            p[..., 0] *= scale
            p[..., 1] *= scale
            p[..., 2] = z - p[..., 0] * cx - p[..., 1] * cy
            out.append(np.ascontiguousarray(p, dtype=np.float32))
        return out

    def layer_sweep(self, E):
        return self.sweep[id(E)]

    def image(self, fill=-7.0):
        return self.devmem.zeros((self.H, self.W), fill)

    def unary_sweep(self, E, out, after_launch=None):
        """bench.py's sweep_unary: every (group, step) of the sweep, device planes, into the H x W image `out`."""
        S, j = self.sweep[id(E)], 0
        for gi, g in enumerate(S.groups):
            base, n = self.devmem.ptr(self.planes_d[gi]), g.plan.num_calls
            for k in range(g.n_steps):
                g.plan.eval_device(base + k * n * 16, self.devmem.ptr(out), self.W * 4, True, 0, planes_on_device=True)
                if after_launch is not None:
                    after_launch(j, gi, g)
                j += 1

    def reference_image(self):
        """The sweep on the PDL-off context, eagerly: the image every other way of issuing it must reproduce."""
        if self._ref is None:
            out = self.image()
            self.unary_sweep(self.R, out)
            self.R.sync()
            assert self.R.overlapped_launch_count == 0
            self._ref = self.devmem.download(out).copy()
        return self._ref

    def oracle(self):
        if self.naive:
            return O.NaiveStereoEnergyOracle(self.imL, self.imR, self.windR, 1e-4, 10.0, 2.0, 0.9, self.D - 1)
        return O.CostVolumeEnergyOracle(self.imL, None, self.vol, None, self.windR, 1e-4, 0.5, self.D - 1)

    def close(self):
        for S in self.sweep.values():
            S.close()
        self.E.close()
        self.R.close()


@pytest.fixture(scope="module")
def side_stream():
    """The caller's stream the contexts under test run on (bench.py: torch's current stream)."""
    import torch
    return torch.cuda.Stream()


@pytest.fixture(scope="module")
def devmem():
    return TorchDeviceMemory()


@pytest.fixture(scope="module")
def expect_overlap():
    """The library always launches with programmatic dependent launch unless LEXP_PDL_OFF=1: the contexts under test must overlap launches."""
    return True


@pytest.fixture(scope="module")
def scene_cache(devmem, side_stream):
    cache = {}
    yield lambda name: cache.get(name) or cache.setdefault(name, Scene(devmem, side_stream, **SCENES[name]))
    for sc in cache.values():
        sc.close()


@pytest.fixture(params=list(SCENES))
def scene(request, scene_cache):
    return scene_cache(request.param)


@pytest.fixture(params=SMALL)
def small_scene(request, scene_cache):
    return scene_cache(request.param)


@pytest.fixture(params=PM_SCENES)
def pm_scene(request, scene_cache):
    return scene_cache(request.param)


def _check_overlapped(E, before, launches, expect_overlap):
    """All launches of a chain but possibly its first carried the programmatic-serialization attribute."""
    n = E.overlapped_launch_count - before
    if expect_overlap:
        assert launches - 1 <= n <= launches, f"{n} of {launches} launches overlapped"
    else:
        assert n == 0


# ---- (a) the unary sweep ----------------------------------------------------------------------------------------------------------
def test_unary_sweep_overlapped_on_a_caller_stream_equals_serialized(scene, expect_overlap):
    """bench.py's unary sweep, eagerly, with set_overlap(True) on the caller's stream: the image of the PDL-off context."""
    ref = scene.reference_image()
    out = scene.image()
    n0, c0 = scene.E.launch_count, scene.E.overlapped_launch_count
    scene.unary_sweep(scene.E, out)
    scene.E.sync()
    assert scene.E.launch_count - n0 == scene.launches
    _check_overlapped(scene.E, c0, scene.launches, expect_overlap)
    assert np.array_equal(scene.devmem.download(out), ref)


def test_unary_sweep_graph_replay_equals_serialized(scene, side_stream):
    """The same sweep captured once into a CUDA graph (as bench.py's capture()) and replayed three times."""
    import torch
    E, ref = scene.E, scene.reference_image()
    out = scene.image()
    g = torch.cuda.CUDAGraph()
    c0 = E.overlapped_launch_count
    with torch.cuda.stream(side_stream):
        with torch.cuda.graph(g):
            E.set_stream(torch.cuda.current_stream().cuda_stream)
            scene.unary_sweep(E, out)
        E.set_stream(side_stream.cuda_stream)
        _check_overlapped(E, c0, scene.launches, True)
        for _ in range(3):
            g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(scene.devmem.download(out), ref)
    del g


def test_unary_sweep_last_writer_wins(small_scene):
    """Consecutive launches of the sweep write the same pixels (the K steps of a group share their targetRects, the sharedRegions
    of successive groups overlap).  Every launch alone, into its own image, composed on the host in issue order, must give the
    serialized sweep's image; the writes must be distinguishable (a reordered write would change the image); and the last step of
    every group is checked against the oracle on sampled cells, over the whole targetRect its launch wrote (of which the sweep's
    image keeps the pixels no later group overwrites)."""
    sc = small_scene
    H, W = sc.H, sc.W
    ref = sc.reference_image()
    S = sc.layer_sweep(sc.R)
    composed = np.full((H, W), -7.0, np.float32)
    last = np.full((H, W), np.nan, np.float32)
    prev = np.full((H, W), np.nan, np.float32)
    writes = np.zeros((H, W), np.int32)
    last_writer = np.full((H, W), -1, np.int64)
    rng = np.random.default_rng(3)
    sampled = {gi: rng.choice(len(g.cells), size=min(2, len(g.cells)), replace=False) for gi, g in enumerate(S.groups)}
    tiles = {}   # (group, cell index) -> (its targetRect in the group's last step, the launch that wrote it)
    launch = 0
    for gi, g in enumerate(S.groups):
        lay = S.layer(g.layer)
        mask = np.zeros((H, W), bool)
        for r in g.cells:
            x, y, w, h = lay.sharedRegions[r]
            mask[y:y + h, x:x + w] = True
        base, n = sc.devmem.ptr(sc.planes_d[gi]), g.plan.num_calls
        for k in range(g.n_steps):
            one = sc.image()
            g.plan.eval_device(base + k * n * 16, sc.devmem.ptr(one), W * 4, True, 0, planes_on_device=True)
            sc.R.sync()
            img = sc.devmem.download(one)
            assert (img[~mask] == -7.0).all(), f"group {gi} step {k} wrote outside its targetRects"
            prev[mask], last[mask] = last[mask], img[mask]
            writes[mask] += 1
            composed[mask] = img[mask]
            last_writer[mask] = launch
            if k == g.n_steps - 1:
                for i in sampled[gi]:
                    x, y, w, h = lay.sharedRegions[g.cells[i]]
                    tiles[(gi, i)] = (img[y:y + h, x:x + w].copy(), launch)
            launch += 1
    assert launch == sc.launches
    assert np.array_equal(composed, ref), "the serialized sweep is not the composition of its launches in issue order"
    multi = writes >= 2
    differ = float((last[multi] != prev[multi]).mean())
    assert multi.any() and differ >= 0.9, f"{multi.sum()} pixels written twice or more, {differ:.3f} of them differ from the write before"

    Or = sc.oracle()
    kept = 0
    for (gi, i), (tile, j) in tiles.items():
        g = S.groups[gi]
        lay = S.layer(g.layer)
        f, t = lay.filterRegions[g.cells[i]], lay.sharedRegions[g.cells[i]]
        assert_costs_close(tile, Or.compute_unary_potential(f, t, sc.planes_h[gi][g.n_steps - 1][i], 0), f"group {gi} cell {g.cells[i]}")
        mine = last_writer[t[1]:t[1] + t[3], t[0]:t[0] + t[2]] == j
        assert np.array_equal(ref[t[1]:t[1] + t[3], t[0]:t[0] + t[2]][mine], tile[mine])
        kept += int(mine.sum())
    assert kept > 0
    print(f"{sc.launches} launches, {multi.sum()} pixels written twice or more ({differ:.3f} differ from the previous write); "
          f"oracle on {len(tiles)} cells, {kept} of their pixels kept in the sweep's image")


# ---- (b) host planes between overlapped launches ------------------------------------------------------------------------------------
def test_host_planes_between_overlapped_launches(scene, expect_overlap):
    """The hazard programmatic dependent launch once exposed: a launch right after the host-to-device copy of its planes read them
    before the copy had landed.  Calls with host planes (each different, into their own image) are interleaved with the overlapped
    device-plane launches of the sweep; none of them may overlap its predecessor, and every image equals its serialized twin."""
    from localexpstereo_b200 import synth
    sc = scene
    every = 8
    n_host = (sc.launches + every - 1) // every
    outs = {}
    for E in (sc.E, sc.R):
        S = sc.layer_sweep(E)
        img, extra = sc.image(), [sc.image() for _ in range(n_host)]   # allocated up front: no synchronisation inside the chain
        c_start = E.overlapped_launch_count

        def host_call(j, gi, g, E=E, S=S, extra=extra):
            if j % every:
                return
            planes = synth.synthetic_planes(S.layer(g.layer).unitRegions, 1, sc.D, 1000 + j)[0][g.cells]
            c0 = E.overlapped_launch_count
            g.plan.eval_device(planes, sc.devmem.ptr(extra[j // every]), sc.W * 4, True, 0)
            assert E.overlapped_launch_count == c0, f"the launch after the plane upload of call {j} overlapped its predecessor"

        sc.unary_sweep(E, img, host_call)
        E.sync()
        # the host-plane launches never overlap; every device-plane launch (but possibly the first) follows a fused launch and does
        _check_overlapped(E, c_start, sc.launches, expect_overlap and E is sc.E)
        outs[id(E)] = [sc.devmem.download(a).copy() for a in [img] + extra]
    got, ref = outs[id(sc.E)], outs[id(sc.R)]
    assert np.array_equal(got[0], ref[0]) and np.array_equal(ref[0], sc.reference_image())
    for j, (a, b) in enumerate(zip(got[1:], ref[1:])):
        assert np.array_equal(a, b), f"host-plane call {j * every}"
        assert (b != -7.0).any()


# ---- (c) the PatchMatch phase -------------------------------------------------------------------------------------------------------
def _pm_labels(S, D):
    """bench.py's initial labels: one per unit of layer 0."""
    from localexpstereo_b200 import synth
    return synth.synthetic_planes(list(S.lm.layers[0].unitRegions), 1, D, 99)[0]


def _assert_state(got, want, what):
    assert np.array_equal(got[0], want[0]), f"{what}: currentCost differs from the serialized run"
    assert np.array_equal(got[1], want[1]), f"{what}: currentLabeling differs from the serialized run"


PM_PREFIX, PM_REPLAYS = 2, 3   # eager iterations 0, 1, then iteration 2 (captured) three times, as bench.py's warm-up + replays


def test_pm_phase_eager_graph_and_native_equal_serialized(pm_scene, side_stream):
    """PMSweep on the caller's stream -- eagerly, and as one captured iteration replayed -- and the library's own schedule object
    (NativePMSweep) under capture: after init and after every iteration the state equals the PDL-off context's, bit for bit."""
    import torch
    from localexpstereo_b200.sweep import NativePMSweep, PMSweep
    sc = pm_scene
    D, IT = sc.D, PM_PREFIX
    its = list(range(PM_PREFIX)) + [IT] * PM_REPLAYS
    Sr = PMSweep(sc.R)
    labels = _pm_labels(Sr, D)
    Sr.begin(); Sr.init(labels[Sr.init_index])
    want = [Sr.get()]
    for it in its:
        Sr.iteration(it, PM_SEED)
        want.append(Sr.get())
    assert sc.R.overlapped_launch_count == 0
    Sr.close()

    E = sc.E
    for name in ("eager", "graph", "native graph"):
        S = NativePMSweep(E) if name == "native graph" else PMSweep(E)
        try:
            S.begin()
            S.init(labels if name == "native graph" else labels[S.init_index])
            _assert_state(S.get(), want[0], f"{name}: init")
            g = None
            for j, it in enumerate(its):
                c0 = E.overlapped_launch_count
                if name == "eager" or j < PM_PREFIX:
                    n = S.iteration(it, PM_SEED)
                    _check_overlapped(E, c0, n, True)
                else:
                    if g is None:
                        g = torch.cuda.CUDAGraph()
                        with torch.cuda.stream(side_stream):
                            with torch.cuda.graph(g):
                                E.set_stream(torch.cuda.current_stream().cuda_stream)
                                n = S.iteration(IT, PM_SEED)
                            E.set_stream(side_stream.cuda_stream)
                        assert n > 0
                        _check_overlapped(E, c0, n, True)
                    with torch.cuda.stream(side_stream):
                        g.replay()
                    torch.cuda.synchronize()
                _assert_state(S.get(), want[j + 1], f"{name}: iteration {j} (index {it})")
            del g
        finally:
            S.close()


def test_pm_replayed_iteration_matches_the_oracle(devmem, side_stream):
    """One captured iteration with planes_out recording, replayed twice: the second replay, re-run by the oracle from the state the
    first one left (pm_get snapshot) with the planes the device recorded, must satisfy the parity protocol of the PatchMatch replay (tests/lexp_replay.py)."""
    import torch
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import PMSweep
    from lexp_testlib import make_scene
    from lexp_replay import check_pm_result, oracle_replay, pointers, recording
    H, W, D, windR, seed, IT = 120, 170, 16, 20, 9, 1
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 4)], [(L.PROP_EXPANSION, 2), (L.PROP_RANDOM, 1)], [(L.PROP_EXPANSION, 2), (L.PROP_RANDOM, 1)]]
    imL, _, volL, _ = make_scene(H, W, D)
    prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
    E = L.CostVolumeEnergy(imL, None, volL, None, prm, D - 1)
    E.set_stream(side_stream.cuda_stream)
    S = PMSweep(E, unit_sizes=[10, 31, 56], proposers=props)
    try:
        S.begin(); S.init(_pm_labels(S, D)[S.init_index])
        S.iteration(0, seed)
        rec, _ = recording(devmem, S, IT, seed)
        g = torch.cuda.CUDAGraph()
        c0 = E.overlapped_launch_count
        with torch.cuda.stream(side_stream):
            with torch.cuda.graph(g):
                E.set_stream(torch.cuda.current_stream().cuda_stream)
                n = S.iteration(IT, seed, planes_out=pointers(devmem, rec))
            E.set_stream(side_stream.cuda_stream)
            _check_overlapped(E, c0, n, True)
            g.replay()
        torch.cuda.synchronize()
        cost_s, lab_s = S.get()
        with torch.cuda.stream(side_stream):
            g.replay()
        torch.cuda.synchronize()
        cost_d, lab_d = S.get()
        rec_host = {k: devmem.download(v) for k, v in rec.items()}
        Or = O.CostVolumeEnergyOracle(imL, None, volL, None, windR, 1e-4, 0.5, D - 1)
        r = oracle_replay(Or, S, cost_s, lab_s, [(False, IT, seed)], [rec_host])
        assert not np.array_equal(cost_d, cost_s)   # the replay did move the state
        check_pm_result(dict(r, cost_d=cost_d, lab_d=lab_d))
        del g
    finally:
        S.close()
        E.close()


# ---- host planes during capture -----------------------------------------------------------------------------------------------------
def test_host_planes_are_refused_during_capture(devmem, side_stream):
    """A call with host planes while the context's stream is being captured is refused with LEXP_ERR_INVALID and enqueues nothing:
    the capture goes on and replays correctly, and the context keeps working with host planes afterwards."""
    import torch
    import localexpstereo_b200 as L
    from localexpstereo_b200 import synth
    H, W, D, windR = 96, 128, 16, 20
    imL = O.synthetic_image(H, W, 42)
    vol = O.synthetic_volume(D, H, W, 1234)
    E = L.CostVolumeEnergy(imL, None, vol, None, L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5), D - 1)
    E.set_stream(side_stream.cuda_stream)
    lay = L.LayerManager(W, H, windR).addLayer(12)
    cells = lay.disjointRegionSets[5]
    plan = E.make_plan([lay.filterRegions[r] for r in cells], [lay.sharedRegions[r] for r in cells])
    planes = synth.synthetic_planes(lay.unitRegions, 1, D, 3)[0][cells]
    ref = np.full((H, W), -7.0, np.float32)
    plan.eval_host(planes, ref)
    d_planes = devmem.upload(planes)
    out, tiles = devmem.zeros((H, W), -7.0), devmem.zeros((plan.target_px,), -7.0)
    try:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(side_stream):
            with torch.cuda.graph(g):
                E.set_stream(torch.cuda.current_stream().cuda_stream)
                with pytest.raises(L.LexpError, match="captured into a CUDA graph"):
                    plan.eval_device(planes, devmem.ptr(out), W * 4, True, 0)
                with pytest.raises(L.LexpError, match="captured into a CUDA graph"):
                    plan.eval_device_tiles(planes, devmem.ptr(tiles), True, 0)
                plan.eval_device(devmem.ptr(d_planes), devmem.ptr(out), W * 4, True, 0, planes_on_device=True)
            E.set_stream(side_stream.cuda_stream)
            g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(devmem.download(out), ref)
        assert (devmem.download(tiles) == -7.0).all()
        out2 = devmem.zeros((H, W), -7.0)
        plan.eval_device(planes, devmem.ptr(out2), W * 4, True, 0)
        E.sync()
        assert np.array_equal(devmem.download(out2), ref)
        del g
    finally:
        plan.close()
        E.close()


# ---- the benchmark's own output -----------------------------------------------------------------------------------------------------
def _run_bench(tmp_path, workload, graph, steps=2, warmup=3):
    import json
    d = tmp_path / f"{workload}_{'graph' if graph else 'eager'}"
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--workload", workload, "--steps", str(steps),
           "--warmup", str(warmup), "--no-cpu-baseline", "--dump-outputs", str(d)] + ([] if graph else ["--no-graph"])
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-4000:]
    assert "capture failed" not in r.stderr, r.stderr[-4000:]
    out = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])
    assert out["config"]["cuda_graph"] is graph
    return {f[:-4]: np.load(d / f) for f in sorted(os.listdir(d))}


def _bench_reproduction(workload, steps, warmup):
    """What bench.py dumps, recomputed in this process on a PDL-off context from the same generators.

    PatchMatch-phase workloads (bench.py:415-437): pms.begin(); pms.init(init_labels[pms.init_index]) with the labels of
    bench.py:422; iterations 0 .. warmup-1 with seed 4321 (:425-426); then iteration `warmup` (IT, :428) 2 + steps times -- the
    two untimed run_pm() calls of :430 and the `steps` timed ones of :433 -- and the dump of the state right after (:435-437).
    The _naive workload (:393-407, :441-447): every sweep writes the same pixels with the same planes, so the dumped image is one
    serialized unary sweep into a zeroed H x W image."""
    import torch
    import bench
    import localexpstereo_b200 as L
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import PMSweep, UnarySweep
    W, H, D, windR = bench.WORKLOADS[workload]
    imL, vol = bench.make_inputs(W, H, D)
    with pdl_off():
        if workload.endswith("_naive"):
            E = L.NaiveStereoEnergy(imL, synth.synthetic_image(H, W, 43), L.Parameters(windR=windR, filterName="GF", filter_param1=bench.EPS), D - 1)
        else:
            E = L.CostVolumeEnergy(imL, None, vol, None, L.Parameters(windR=windR, filterName="GF", filter_param1=bench.EPS, th_col=bench.TH_COL), D - 1)
    try:
        if workload.endswith("_naive"):
            unary = UnarySweep(E, unit_sizes=[5, 15, 25])
            planes_d = [torch.from_numpy(p).cuda() for p in bench.all_planes(unary, D)]
            cost_d = torch.zeros((H, W), dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            for gi, g in enumerate(unary.groups):
                base, n = planes_d[gi].data_ptr(), g.plan.num_calls
                for k in range(g.n_steps):
                    g.plan.eval_device(base + k * n * 16, cost_d.data_ptr(), W * 4, True, 0, planes_on_device=True)
            E.sync()
            unary.close()
            assert E.overlapped_launch_count == 0
            return {"unary_cost": cost_d.cpu().numpy()}
        pms = PMSweep(E)
        pms.begin()
        init_labels = synth.synthetic_planes([pms.lm.layers[0].unitRegions[i] for i in range(len(pms.lm.layers[0].unitRegions))], 1, D, 99)[0]
        pms.init(init_labels[pms.init_index])
        for it in range(warmup):
            pms.iteration(it, PM_SEED)
        for _ in range(2 + steps):
            pms.iteration(warmup, PM_SEED)
        cost, lab = pms.get()
        pms.close()
        assert E.overlapped_launch_count == 0
        return {"current_cost": cost, "current_labeling": lab}
    finally:
        E.close()


@pytest.mark.parametrize("workload", ["tiny_450x375x64_r20", "middv2_cones_shape_450x375x64_naive"])
def test_bench_graph_and_eager_outputs_equal_a_serialized_reproduction(tmp_path, workload):
    """bench.py as a subprocess, with and without its CUDA graph: the graph is really used, both dumps are identical, and they
    equal the same sequence run here on a PDL-off context."""
    steps, warmup = 2, 3
    graph = _run_bench(tmp_path, workload, True, steps, warmup)
    eager = _run_bench(tmp_path, workload, False, steps, warmup)
    want = _bench_reproduction(workload, steps, warmup)
    assert sorted(graph) == sorted(eager) == sorted(want)
    for k in want:
        assert np.array_equal(graph[k], eager[k]), f"{k}: graph and eager runs differ"
        assert np.array_equal(graph[k], want[k].astype(np.float32)), f"{k}: the benchmark's output differs from the serialized reproduction"
