"""Every PatchMatch step of the device against the oracle's update of the SAME state.

tests/test_gpu_pm.py replays the device's planes in the numpy oracle on the oracle's own state, which drifts from the device's at
FP32 / FP64 cost ties, so it needs budgets.  Here every step starts from the device's own pre-step state (pm_get) and is certified
without a budget (Rig.certify):
  (P) proposal: the oracle's proposer (oracle.pm_proposal) on the device's pre-step labeling, with the launch's random stream, gives
      the plane the step recorded -- bit for bit for lists and ExpansionProposer; RandomProposer within 2e-6 relative / 1e-6 absolute
      (CUDA's FP64 sin / cos against glibc's), its fourth component bit for bit;
  (U) update: nothing outside the group's targetRects changes; inside, post = (pre_cost > q) ? (q, plane) : pre bit for bit (a NaN
      cost never updates), or (q, plane) unconditionally for an initialisation.  q is the PatchMatch instantiation's own proposal
      cost: the recorded planes run as an initialisation on a twin context (same inputs, its own state and schedule);
  (Q) q against the FP64 C oracle (oracle.c_oracle, which tests/test_ref_pin.py pins to the reference): 1e-4 relative, the exact
      COST_FOR_INVALID mask and the NaN pattern;
  (I) q equals the unary instantiation's cost of the same planes (Plan.eval_device: image output, with the check) bit for bit --
      the graph-cut steps take their proposal costs from that instantiation.
Steps are issued one at a time with a synchronisation in between; the final state must equal the twin's uninterrupted sweep bit
for bit (tests/test_gpu_launch_chains.py shows that overlapped launches equal serialized ones).

Pixel tags: the fourth plane component v enters the cost only as 0 * v and through isfinite, and RandomProposer copies it.  With
v = y * W + x in every pixel after the initialisation, a proposal names the pixel it was drawn from.
(Sorted after the graph-cut tests and before the large-size tests.)"""
import time

import numpy as np
import pytest

from oracle import c_oracle
from oracle import lexp_oracle as O
from lexp_testlib import TorchDeviceMemory, assert_costs_close, bits, make_scene, seeded_labels

pytestmark = pytest.mark.gpu

INVALID = np.float32(O.COST_FOR_INVALID)


@pytest.fixture(scope="module")
def devmem():
    return TorchDeviceMemory()


def ulps(a, b):
    """Distance in units in the last place of two float32 arrays of the same sign."""
    return np.abs(bits(a).astype(np.int64) - bits(b).astype(np.int64))


class Tally:
    def __init__(self):
        self.steps = self.exact = self.n_exact = self.random = self.n_random = self.random_same = 0
        self.named = self.n_named = 0
        self.worst_q = 0.0
        self.instantiations_agree = True
        self.t_oracle = self.t_step = 0.0

    def line(self, what):
        frac = self.random_same / self.n_random if self.n_random else 1.0
        return (f"{what}: {self.steps} steps certified; proposals: list / Expansion bit-identical {self.exact} of {self.n_exact}, "
                f"Random within tolerance {self.random} of {self.n_random} ({frac:.4f} bit-identical); source pixels named by their tag "
                f"{self.named} of {self.n_named}; worst q err vs the FP64 oracle {self.worst_q:.2e}; (I) PM = unary instantiation: "
                f"{'held' if self.instantiations_agree else 'FAILED'}; {self.t_step:.1f} s certifying, {self.t_oracle:.1f} s of it in the C oracle")


class Rig:
    """The context under test E and its twin Eq on the same inputs, a PMSweep on each, the FP64 C oracle of the view and page-locked
    buffers for the states."""

    def __init__(self, devmem, imL, imR, volL, volR, windR, units, proposers, mode=0, MIN=0.0, MAX=None, vol_host=None):
        import localexpstereo_b200 as L
        from localexpstereo_b200.sweep import PMSweep
        self.L, self.dm, self.mode = L, devmem, mode
        vol = volR if mode else volL
        D = int(vol.shape[0])
        self.MAX = float(D - 1 if MAX is None else MAX)
        self.MIN = float(MIN)
        prm = L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)
        self.E, self.Eq = [L.CostVolumeEnergy(imL, imR, volL, volR, prm, self.MAX, self.MIN) for _ in range(2)]
        self.H, self.W = self.E.height, self.E.width
        self.S, self.Sq = [PMSweep(E, unit_sizes=units, proposers=proposers, mode=mode) for E in (self.E, self.Eq)]
        self.C = c_oracle.COracle(self.H, self.W, D, windR, 1e-4, 0.5, self.MAX, self.MIN)
        self.C.set_image(mode, imR if mode else imL)
        self.C.set_volume(mode, vol if vol_host is None else vol_host)
        self.buf = {}
        for k in ("pre", "post", "q"):
            self.buf[k] = (np.empty((self.H, self.W), np.float32), np.empty((self.H, self.W, 4), np.float32))
            for a in self.buf[k]:
                L.host_register(a)
        self.owner = {}
        self.tags = (np.arange(self.H, dtype=np.float32)[:, None] * np.float32(self.W) + np.arange(self.W, dtype=np.float32)[None, :])
        self.tagged = self.tag_check_pending = False
        self.T = Tally()

    def close(self):
        for a in (x for pair in self.buf.values() for x in pair):
            self.L.host_unregister(a)
        for S in (self.S, self.Sq):
            S.close()
        for E in (self.E, self.Eq):
            E.close()
        self.C.close()

    def get(self, E, key=None):
        if key is None:
            return E.pm_get(self.mode)
        return E.pm_get(self.mode, out_cost=self.buf[key][0], out_labeling=self.buf[key][1])

    def tag(self, E):
        """v = y * W + x in every pixel of E's state (exact: below 2^24), the costs unchanged.  Tagging the state under test also
        makes its next certified step check that the tags leave the proposal costs unchanged."""
        assert self.H * self.W <= 1 << 24
        c, l = self.get(E)
        l[..., 3] = self.tags
        E.pm_begin(self.mode, c, l)
        if E is self.E:
            self.tagged = self.tag_check_pending = True

    def owner_of(self, targets):
        """[H][W] int: the call whose targetRect holds the pixel, -1 outside all of them (they must be disjoint)."""
        key = tuple(map(tuple, targets))
        if key not in self.owner:
            o = np.full((self.H, self.W), -1, np.int64)
            for i, (x, y, w, h) in enumerate(targets):
                assert (o[y:y + h, x:x + w] == -1).all(), "targetRects of one step overlap"
                o[y:y + h, x:x + w] = i
            self.owner[key] = o
        return self.owner[key]

    def twin_q(self, qplan, d_planes=None, planes=None):
        """The PatchMatch instantiation's cost of the planes in every target pixel: an initialisation step on the twin."""
        self.Eq.pm_reset_sync()
        if d_planes is not None:
            qplan.pm_step(0, self.L.PROP_LIST, planes=d_planes, planes_on_device=True, init=True, mode=self.mode)
        else:
            qplan.pm_step(0, self.L.PROP_LIST, planes=planes, init=True, mode=self.mode)
        self.Eq.sync()
        return self.get(self.Eq, "q")

    def certify(self, g, qplan, kind, m=0, seed=0, step_index=0, init=False, planes=None, sync=None):
        """One step of the GroupPlan g (qplan: the twin's plan of the same cells) checked by (P), (U), (Q) and (I) of the module docstring.
        Returns (pre, post, inside, q): the states are views of buffers the next step overwrites; inside marks the target pixels,
        q holds their proposal costs."""
        L, E, dm, T = self.L, self.E, self.dm, self.T
        t0 = time.perf_counter()
        plan, units, targets, filters, ids = g.plan, g.units, g.targets, g.filters, g.ids
        n = plan.num_calls
        assert len(units) == n and (kind == L.PROP_LIST) == (planes is not None)
        pre_c, pre_l = self.get(E, "pre")
        rec = dm.zeros((n, 4), fill=np.nan)
        plan.pm_step(step_index, kind, m, seed, planes=planes, d_planes_out=dm.ptr(rec), init=init, mode=self.mode, **(sync or {}))
        E.sync()
        post_c, post_l = self.get(E, "post")
        used = np.array(dm.download(rec), np.float32)
        # (P)
        for i, u in enumerate(units):
            if kind == L.PROP_LIST:
                assert np.array_equal(bits(used[i]), bits(planes[i])), f"(P) call {i}: recorded {used[i]}, listed {planes[i]}"
                T.n_exact += 1; T.exact += 1
                continue
            st = O.pm_rng_state(seed, ids[i])
            mine = O.pm_proposal(kind, m, st, pre_l, u, self.MIN, self.MAX)
            if self.tagged:
                nn = O.CvRNG(st).uniform_int(0, u[2] * u[3])
                sx, sy = u[0] + nn % u[2], u[1] + nn // u[2]
                T.n_named += 1
                T.named += int(pre_l[sy, sx, 3] == self.tags[sy, sx] and used[i, 3] == self.tags[sy, sx])
            if kind == L.PROP_EXPANSION:
                T.n_exact += 1
                assert np.array_equal(bits(used[i]), bits(mine)), f"(P) Expansion, cell {ids[i]} unit {u}: device {used[i]}, oracle {mine}"
                T.exact += 1
            else:
                T.n_random += 1
                assert bits(used[i])[3] == bits(mine)[3] and np.allclose(used[i], mine, rtol=2e-6, atol=1e-6), \
                    f"(P) Random m={m}, cell {ids[i]} unit {u}: device {used[i]!r}, oracle {mine!r}"
                T.random += 1
                T.random_same += int(np.array_equal(bits(used[i]), bits(mine)))
        # q: the PatchMatch instantiation, on the twin
        q_c, q_l = self.twin_q(qplan, d_planes=dm.ptr(rec))
        own = self.owner_of(targets)
        inside = own >= 0
        plane_px = used[own[inside]]
        q = q_c[inside]
        assert np.array_equal(bits(q_l[inside]), bits(plane_px)), "the twin's initialisation did not write the recorded planes"
        if self.tag_check_pending:   # v enters the cost as 0 * v only: the same planes with v = 0 cost the same, bit for bit
            self.tag_check_pending = False
            flat = used.copy()
            flat[:, 3] = 0.0
            q0 = self.twin_q(qplan, planes=flat)[0][inside]
            assert np.array_equal(bits(q0), bits(q)), "pixel tags changed a proposal cost"
        # (U)
        pc, pl = pre_c[inside], pre_l[inside]
        upd = np.ones(q.shape, bool) if init else pc > q
        assert np.array_equal(bits(post_c[inside]), bits(np.where(upd, q, pc))), \
            f"(U) cost: {int((bits(post_c[inside]) != bits(np.where(upd, q, pc))).sum())} target pixels differ from the rule"
        assert np.array_equal(bits(post_l[inside]), bits(np.where(upd[:, None], plane_px, pl))), "(U) label differs from the rule"
        assert np.array_equal(bits(post_c[~inside]), bits(pre_c[~inside])) and np.array_equal(bits(post_l[~inside]), bits(pre_l[~inside])), \
            "(U) a pixel outside the step's targetRects changed"
        # (Q)
        t1 = time.perf_counter()
        ref = np.zeros((self.H, self.W), np.float32)
        self.C.unary_batch(self.mode, filters, targets, used, ref, with_check=True)
        T.t_oracle += time.perf_counter() - t1
        r = ref[inside]
        nan = np.isnan(r)
        assert np.array_equal(nan, np.isnan(q)), f"(Q) NaN pattern differs at {int((nan != np.isnan(q)).sum())} pixels"
        T.worst_q = max(T.worst_q, assert_costs_close(q[~nan], r[~nan], f"(Q) step kind {kind} m {m}"))
        # (I)
        img = dm.zeros((self.H, self.W), fill=np.nan)
        plan.eval_device(dm.ptr(rec), dm.ptr(img), self.W * 4, with_check=True, mode=self.mode, planes_on_device=True)
        E.sync()
        ev = np.array(dm.download(img), np.float32)[inside]
        same = bits(ev) == bits(q)
        if not same.all():
            T.instantiations_agree = False
            bad = ~same
            raise AssertionError(f"(I) the PatchMatch and unary instantiations differ at {int(bad.sum())} of {bad.size} pixels, up to "
                                 f"{int(ulps(ev[bad], q[bad]).max())} ulps (e.g. {ev[bad][0]!r} vs {q[bad][0]!r})")
        T.steps += 1
        T.t_step += time.perf_counter() - t0
        return (pre_c, pre_l), (post_c, post_l), inside, q

    # ---- the sweep's own walk (PMSweep.init / iteration_by_group), one step at a time ----------------------------------------------
    def init(self, labels, certify=True):
        def issue(g, steps):
            ((k, kind, _, _, sync),) = steps
            if certify:
                self.certify(g, self.Sq.init_plan, kind, planes=np.asarray(labels, np.float32), init=True, sync=sync)
            else:
                g.plan.pm_step(k, kind, planes=labels, init=True, mode=self.mode, **sync)
        for _ in self.S.walk(None, 0, issue):
            pass

    def iteration(self, it, seed, certify=lambda li: True, snap_layer=None):
        """One iteration of the sweep under test; steps of the layers `certify` selects are certified.  Returns the state at the end
        of layer snap_layer (None: not taken)."""
        S, snap = self.S, None
        twin = {(g.layer, g.group): g.plan for g in self.Sq.groups}

        def issue(g, steps):
            for k, kind, m, sd, sync in steps:
                if certify(g.layer):
                    self.certify(g, twin[(g.layer, g.group)], kind, m, sd, k, sync=sync)
                else:
                    g.plan.pm_step(k, kind, m, sd, mode=self.mode, **sync)
        for n, _ in enumerate(S.walk(it, seed, issue)):
            li = S.schedule[n][0]
            if li == snap_layer and (n + 1 == len(S.schedule) or S.schedule[n + 1][0] != li):
                snap = self.get(self.E)
        return snap

    def twin_reference(self, labels, seed, upto, tag=False):
        """The twin's uninterrupted sweep (PMSweep.init / iteration_by_group): the state after the initialisation (upto = None) or
        at the end of layer upto[1] of iteration upto[0], iterations 0 .. upto[0] run in full."""
        Sq = self.Sq
        Sq.begin()
        Sq.init(labels)
        if tag:
            self.tag(self.Eq)
        if upto is None:
            return self.get(self.Eq)
        ref = None
        for it in range(upto[0] + 1):
            for n, _ in enumerate(Sq.iteration_by_group(it, seed)):
                li = Sq.schedule[n][0]
                if (it, li) == tuple(upto) and (n + 1 == len(Sq.schedule) or Sq.schedule[n + 1][0] != li):
                    ref = self.get(self.Eq)
        return ref


def assert_same_state(a, b, what):
    assert np.array_equal(bits(a[0]), bits(b[0])), f"{what}: currentCost differs at {int((bits(a[0]) != bits(b[0])).sum())} pixels"
    assert np.array_equal(bits(a[1]), bits(b[1])), f"{what}: currentLabeling differs"


def run_sweep(R, labels, iterations, seed, tag=True, what="scene"):
    """The twin uninterrupted, then the sweep under test step by step with every step certified (the initialisation included);
    the final states must be bit-identical."""
    ref = R.twin_reference(labels, seed, (iterations - 1, len(R.S.unit_sizes) - 1), tag=tag)
    R.E.pm_begin(R.mode)
    R.init(labels)
    if tag:
        R.tag(R.E)
    for it in range(iterations):
        R.iteration(it, seed)
    assert_same_state(R.get(R.E), ref, f"{what}: step by step against uninterrupted")
    print(R.T.line(what))
    return R.T


# ---- designed scenes (small) -------------------------------------------------------------------------------------------------------------
def small_rig(devmem, H, W, D, windR, units, proposers, mode=0, seed=0, MIN=0.0, MAX=None):
    imL, imR, volL, volR = make_scene(H, W, D, seed=seed)
    return Rig(devmem, imL, imR, volL, volR, windR, units, proposers, mode, MIN, MAX)


def scene_tags(devmem, mode=0):
    """A ragged image (the last unit of every row and column is narrower), two layers, Expansion and Random, two iterations, the
    state tagged after the initialisation: every proposal names its source pixel."""
    import localexpstereo_b200 as L
    H, W, D = 67, 89, 12
    R = small_rig(devmem, H, W, D, 12, [7, 19], [[(L.PROP_EXPANSION, 2), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]],
                  mode, seed=3)
    try:
        for lay in R.S.lm.layers:
            us = lay.unitRegions
            assert min(u[2] for u in us) < lay.regionUnitSize and min(u[3] for u in us) < lay.regionUnitSize, "the image should be ragged"
        T = run_sweep(R, seeded_labels(R.S, 21), 2, 5, what=f"pixel tags, mode {mode}")
        assert T.n_exact > 300 and T.n_random > 300 and T.named > 0
        return T
    finally:
        R.close()


def scene_update_edges(devmem, mode=0):
    """PROP_LIST steps on designed states: ties, the next float above q, NaN, +inf and COST_FOR_INVALID against an invalid plane, a
    NaN plane."""
    import localexpstereo_b200 as L
    H, W, D = 40, 56, 12
    R = small_rig(devmem, H, W, D, 12, [8], [[(L.PROP_EXPANSION, 1)]], mode, seed=8)
    try:
        S = R.S
        R.Eq.pm_begin(mode)
        (_, _, g, _), (_, _, gq, _) = S.schedule[5], R.Sq.schedule[5]
        n = g.plan.num_calls
        old = np.zeros((H, W, 4), np.float32)
        old[..., 2] = 3.0
        rs = np.random.default_rng(mode)
        good = np.stack([[rs.uniform(-0.05, 0.05), rs.uniform(-0.05, 0.05), rs.uniform(4, 7), 7.0] for _ in range(n)]).astype(np.float32)
        far = np.tile(np.float32([0, 0, -50, 1]), (n, 1))
        nanp = np.tile(np.float32([np.nan, 0, 5, 2]), (n, 1))

        def step(cost, planes):
            R.E.pm_reset_sync()
            R.E.pm_begin(mode, cost, old)
            pre, post, inside, q = R.certify(g, gq.plan, L.PROP_LIST, planes=planes)
            changed = (bits(post[0]) != bits(pre[0])) | (bits(post[1]) != bits(pre[1])).any(axis=2)
            return inside, q, changed

        inf = np.full((H, W), np.inf, np.float32)
        inside, q, changed = step(inf, good)                  # +inf: every target pixel takes the plane
        assert np.array_equal(changed, inside) and (q != INVALID).all()
        qimg = np.ones((H, W), np.float32)
        qimg[inside] = q
        assert not step(qimg, good)[2].any(), "a tie (cur == q) must not update"
        _, _, changed = step(np.nextafter(qimg, np.float32(np.inf)), good)
        assert np.array_equal(changed, inside), "cur = nextafter(q, +inf) must update every target pixel"
        assert not step(np.full((H, W), np.nan, np.float32), good)[2].any(), "a NaN current cost must never update"
        _, q, changed = step(inf, far)
        assert (q == INVALID).all() and np.array_equal(changed, inside), "+inf against COST_FOR_INVALID must update"
        assert not step(np.full((H, W), INVALID, np.float32), far)[2].any(), "COST_FOR_INVALID against COST_FOR_INVALID must not update"
        mixed = np.where(rs.random((H, W)) < 0.5, np.float32(np.inf), np.float32(0.5))
        step(mixed, nanp)                                      # a NaN plane: whatever q the oracle gives it, the rule holds
        print(R.T.line(f"update edges, mode {mode}"))
    finally:
        R.close()


def scene_min_max(devmem, mn, mx):
    """MIN_DISPARITY != 0 or MAX_DISPARITY != D - 1: the generic sampler inside the PatchMatch kernel and RandomProposer's clamps."""
    import localexpstereo_b200 as L
    H, W, D = 48, 70, 16
    R = small_rig(devmem, H, W, D, 12, [8, 20], [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 3)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)]],
                  seed=77, MIN=mn, MAX=mx)
    try:
        run_sweep(R, seeded_labels(R.S, 13), 1, 9, what=f"MIN {mn}, MAX {mx}")
    finally:
        R.close()


def scene_many_items(devmem):
    """Every layer-1 cell cut into >= 32 work items (LEXP_TILE_OH = 8, set by the caller before the contexts exist): the proposal
    hand-over through the cell's ticket, ready flag and plane."""
    import localexpstereo_b200 as L
    H, W, D = 140, 150, 12
    R = small_rig(devmem, H, W, D, 12, [19, 64], [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]],
                  seed=4)
    try:
        items = [g.plan.num_items / g.plan.num_calls for g in R.S.groups if g.layer == 1]
        assert min(items) >= 32, items
        run_sweep(R, seeded_labels(R.S, 17), 1, 3, what=f"{min(items):.0f} work items per layer-1 cell")
    finally:
        R.close()


def scene_random_m(devmem, mode=1):
    """Direct RandomProposer steps with m = 0, 1 and 120 (the C-ABI's bound: exp2f(-121) is still a normal float) on a tagged state,
    with the random streams of the sweep's three RandomProposer steps of iteration 0 (seed 8)."""
    import localexpstereo_b200 as L
    H, W, D = 44, 60, 12
    R = small_rig(devmem, H, W, D, 12, [8], [[(L.PROP_RANDOM, 3)]], mode, seed=6)
    try:
        S = R.S
        R.Eq.pm_begin(mode)
        R.E.pm_begin(mode)
        R.init(seeded_labels(S, 31))
        R.tag(R.E)
        for (li, gi, g, _), (_, _, gq, _) in list(zip(S.schedule, R.Sq.schedule))[:8]:
            R.E.pm_reset_sync()
            for (k, kind, _, sd), m in zip(S.group_steps(li, gi, 0, 8), (0, 1, 120)):
                R.certify(g, gq.plan, kind, m, sd, k)
        print(R.T.line(f"Random at m = 0, 1, 120, mode {mode}"))
        assert R.T.n_random > 80 and R.T.named > 0
    finally:
        R.close()


# ---- tests: designed scenes --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [0, 1])
def test_pixel_tags_name_every_source_pixel(devmem, mode):
    scene_tags(devmem, mode)


@pytest.mark.parametrize("mode", [0, 1])
def test_update_rule_at_its_edges(devmem, mode):
    scene_update_edges(devmem, mode)


@pytest.mark.parametrize("mn,mx", [(-4.0, 11.0), (0.0, 9.0)])
def test_nonzero_min_and_short_max_disparity(devmem, mn, mx):
    scene_min_max(devmem, mn, mx)


def test_many_work_items_per_cell(devmem, monkeypatch):
    monkeypatch.setenv("LEXP_TILE_OH", "8")
    scene_many_items(devmem)


def test_random_proposer_at_the_ends_of_m(devmem):
    scene_random_m(devmem, mode=1)


# ---- at scale -----------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bench_rig(devmem):
    """bench.py's PatchMatch-phase workload: 2048 x 1536 x 256, windR 20, V3_PROPOSERS_DEVICE, initial labels of bench.py (seed 99),
    the volume drawn on the device (torch.rand, seed 1234) and copied to the host for the C oracle (3.2 GB)."""
    import torch
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import V3_PROPOSERS_DEVICE
    W, H, D, windR = 2048, 1536, 256, 20
    imL = synth.synthetic_image(H, W, 42)
    vol = torch.rand((D, H, W), generator=torch.Generator(device="cuda").manual_seed(1234), device="cuda", dtype=torch.float32)
    torch.cuda.synchronize()
    R = Rig(devmem, imL, None, vol, None, windR, None, V3_PROPOSERS_DEVICE, vol_host=vol.cpu().numpy())
    del vol
    torch.cuda.empty_cache()
    units = R.S.lm.layers[0].unitRegions
    labels = synth.synthetic_planes([units[i] for i in range(len(units))], 1, D, 99)[0][R.S.init_index]
    yield R, labels
    R.close()


BENCH_SEED = 4321
BENCH_REPLAYED = 3   # bench.py's default --warmup: the iteration index it captures and replays


@pytest.mark.parametrize("it,layer", [(None, None)] + [(it, li) for it in (0, BENCH_REPLAYED) for li in range(3)])
def test_every_step_of_the_benchmark_workload(bench_rig, it, layer):
    """The initialisation (it = None), or every step of one layer of iteration `it` after iterations 0 .. it - 1 and the layer's
    predecessors ran uninterrupted; the state tagged after the initialisation on both contexts.  The state at the end of the layer
    must equal the twin's uninterrupted sweep."""
    R, labels = bench_rig
    R.T, R.tagged, R.tag_check_pending = Tally(), False, False
    t0 = time.perf_counter()
    ref = R.twin_reference(labels, BENCH_SEED, None if it is None else (it, layer), tag=True)
    R.E.pm_begin(0)
    R.init(labels, certify=it is None)
    R.tag(R.E)
    if it is None:
        state = R.get(R.E)
    else:
        for i in range(it):
            R.iteration(i, BENCH_SEED, certify=lambda li: False)
        state = R.iteration(it, BENCH_SEED, certify=lambda li: li == layer, snap_layer=layer)
    what = "benchmark workload, " + ("initialisation" if it is None else f"iteration {it}, layer {layer}")
    assert_same_state(state, ref, what)
    print(R.T.line(what) + f"; {time.perf_counter() - t0:.1f} s in all")
    assert R.T.steps == (1 if it is None else 16 * (9 if layer == 0 else 3))


def scene_at_size(devmem, W, H, D, windR, mode, seed):
    """Two iterations of V3_PROPOSERS_DEVICE on a synthetic scene, every step certified, the state tagged after the initialisation."""
    from localexpstereo_b200.sweep import V3_PROPOSERS_DEVICE
    imL, imR, volL, volR = make_scene(H, W, D, seed=seed)
    R = Rig(devmem, imL, imR if mode else None, volL, volR if mode else None, windR, None, V3_PROPOSERS_DEVICE, mode)
    try:
        t0 = time.perf_counter()
        run_sweep(R, seeded_labels(R.S, seed), 2, 1000 + seed, what=f"{W} x {H} x {D}, windR {windR}, mode {mode}")
        print(f"  {time.perf_counter() - t0:.1f} s in all")
    finally:
        R.close()


def test_every_step_of_the_r16_instantiation(devmem):
    scene_at_size(devmem, 960, 544, 96, 32, 0, 5)


def test_every_step_of_the_generic_radius_right_view(devmem):
    scene_at_size(devmem, 437, 291, 40, 12, 1, 6)
