"""Every PatchMatch step of the device against the oracle's update of the SAME state, for both energies: the cost-volume energy
(tests/test_gpu_zz_pm_steps.py, tests/test_gpu_zz_lean.py, tests/test_gpu_ransac.py) and the image-based energy of `-mode MiddV2`
(tests/naive_pm_checks.py).

A whole-run replay (tests/test_gpu_pm.py) runs the oracle on its own state, which drifts from the device's at FP32 / FP64 cost ties,
so it needs budgets.  Here every step starts from the device's own pre-step state (pm_get) and is certified without a budget
(Rig.certify):
  (P) proposal: the oracle's proposer (oracle.pm_proposal) on the device's pre-step labeling, with the launch's random stream, gives
      the plane the step recorded -- bit for bit for lists, ExpansionProposer and RansacProposer; RandomProposer within 2e-6
      relative / 1e-6 absolute (CUDA's FP64 sin / cos against glibc's), its fourth component bit for bit;
  (U) update: nothing outside the group's targetRects changes; inside, post = (pre_cost > q) ? (q, plane) : pre bit for bit (a NaN
      cost never updates), or (q, plane) unconditionally for an initialisation.  q is the PatchMatch instantiation's own proposal
      cost: the recorded planes run as an initialisation on a twin context (same inputs, its own state and schedule);
  (Q) q against an oracle of the energy, with the exact COST_FOR_INVALID mask.  Guided filter ("GF"): 1e-4 relative; cost-volume
      energy: the FP64 C oracle (oracle.c_oracle, which tests/test_ref_pin.py pins to the reference) on every target pixel, and the
      NaN pattern; image-based energy: the numpy oracle on q_cells cells of every step, drawn from the rig's own random stream.
      The bilateral filter ("BL" / "BF") and none (""), under the rules of tests/filter_checks.compare (NaN pattern exact, "" bit for
      bit, bilateral |d| <= 1e-5 max(sum w |p|, 1e-3)): cost-volume energy on every target pixel against
      COracle.filter_unary_batch (which tests/test_filter_c_oracle.py pins to oracle/filter_oracle.py), image-based energy on q_cells
      cells against oracle/filter_oracle.py;
  (I) q equals the unary instantiation's cost of the same planes (Plan.eval_device: image output, with the check) bit for bit --
      the graph-cut steps take their proposal costs from that instantiation.
run_sweep issues the steps one at a time with a synchronisation in between; the final state must equal the twin's uninterrupted sweep
bit for bit (tests/test_gpu_launch_chains.py shows that overlapped launches equal serialized ones).

Pixel tags (cost-volume energy only): the fourth plane component v enters that cost only as 0 * v and through isfinite, and
RandomProposer copies it.  With v = y * W + x in every pixel after the initialisation, a proposal names the pixel it was drawn from.
The same holds with the bilateral filter and none ("BL" / ""), whose weights come from the guide alone.  In the image-based energy v
shifts the warp, so it changes the cost: tagging that state raises."""
import time

import numpy as np

from oracle import c_oracle
from oracle import lexp_oracle as O
import filter_checks as FC
from lexp_testlib import assert_costs_close, bits

NAIVE_FILTERS = ("GF", "BF", "")
CV_FILTERS = ("GF", "BL", "")


def ulps(a, b):
    """Distance in units in the last place of two float32 arrays of the same sign."""
    return np.abs(bits(a).astype(np.int64) - bits(b).astype(np.int64))


class Tally:
    def __init__(self):
        self.steps = self.exact = self.n_exact = self.ransac = self.random = self.n_random = self.random_same = 0
        self.named = self.n_named = self.q_cells = 0
        self.worst_q = 0.0
        self.t_oracle = self.t_step = 0.0

    def line(self, what):
        frac = self.random_same / self.n_random if self.n_random else 1.0
        return (f"{what}: {self.steps} steps certified; proposals: list / Expansion / RANSAC bit-identical {self.exact} of {self.n_exact} "
                f"(RANSAC {self.ransac}), Random within tolerance {self.random} of {self.n_random} ({frac:.4f} bit-identical); source pixels "
                f"named by their tag {self.named} of {self.n_named}; (Q) {self.q_cells} cells, worst q err vs the oracle {self.worst_q:.2e}; "
                f"(I) PM = unary instantiation: held; {self.t_step:.1f} s certifying, {self.t_oracle:.1f} s of it in the (Q) oracle")


class Rig:
    """The context under test E and its twin Eq on the same inputs, a PMSweep on each, the oracle of the energy for (Q) and
    page-locked buffers for the states.  naive=False: CostVolumeEnergy on (imL, imR, volL, volR) (vol_host: a host copy of the view's
    volume for the C oracle, when that volume is on the device); naive=True: NaiveStereoEnergy on (imL, imR) with the parameters of
    `-mode MiddV2` (volL, volR unused, MAX required), (Q) on q_cells cells per step drawn with np.random.default_rng(seed).
    filter: the contexts' filterName -- "GF" (the guided filter, eps 1e-4), "BL" (cost volume) / "BF" (image-based): the bilateral
    filter with sig2, "": none."""

    def __init__(self, devmem, imL, imR, volL, volR, windR, units, proposers, mode=0, MIN=0.0, MAX=None, vol_host=None, naive=False,
                 q_cells=4, seed=0, filter="GF", sig2=10.0):
        import localexpstereo_b200 as L
        from localexpstereo_b200.sweep import PMSweep
        self.L, self.dm, self.mode, self.naive = L, devmem, mode, naive
        self.MIN = float(MIN)
        assert filter in (NAIVE_FILTERS if naive else CV_FILTERS), f"filterName {filter!r}"
        self.filter, self.windR, self.sig2 = filter, windR, sig2
        if naive:
            from naive_pm_checks import MIDDV2_LAMBDA, middv2_params
            prm = middv2_params(windR) if filter == "GF" else L.Parameters(lambda_=MIDDV2_LAMBDA, windR=windR, filterName=filter,
                                                                           filter_param1=sig2)
            self.MAX = float(MAX)
            self.E, self.Eq = [L.NaiveStereoEnergy(imL, imR, prm, self.MAX, self.MIN) for _ in range(2)]
            if filter == "GF":
                self.Or = O.NaiveStereoEnergyOracle(imL, imR, windR, 1e-4, prm.th_col, prm.th_grad, prm.alpha, self.MAX, self.MIN)
            else:
                from oracle.filter_oracle import FilteredEnergyOracle
                self.Or = FilteredEnergyOracle.naive(imL, imR, windR, sig2, prm.th_col, prm.th_grad, prm.alpha, self.MAX, self.MIN,
                                                     bilateral=filter == "BF")
            self.rng, self.q_cells = np.random.default_rng(seed), q_cells
        else:
            vol = volR if mode else volL
            D = int(vol.shape[0])
            self.MAX = float(D - 1 if MAX is None else MAX)
            prm = L.Parameters(windR=windR, filterName=filter, filter_param1=1e-4 if filter == "GF" else sig2, th_col=0.5)
            self.E, self.Eq = [L.CostVolumeEnergy(imL, imR, volL, volR, prm, self.MAX, self.MIN) for _ in range(2)]
        self.H, self.W = self.E.height, self.E.width
        self.S, self.Sq = [PMSweep(E, unit_sizes=units, proposers=proposers, mode=mode) for E in (self.E, self.Eq)]
        if not naive:
            self.C = c_oracle.COracle(self.H, self.W, D, windR, 1e-4, 0.5, self.MAX, self.MIN)
            self.C.set_image(mode, imR if mode else imL)
            self.C.set_volume(mode, vol if vol_host is None else vol_host)
        self.buf = {}
        for k in ("pre", "post", "q"):
            self.buf[k] = (np.empty((self.H, self.W), np.float32), np.empty((self.H, self.W, 4), np.float32))
            for a in self.buf[k]:
                L.host_register(a)
        self.owner = {}
        self.fq = None
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
        if not self.naive:
            self.C.close()

    def get(self, E, key=None):
        if key is None:
            return E.pm_get(self.mode)
        return E.pm_get(self.mode, out_cost=self.buf[key][0], out_labeling=self.buf[key][1])

    def tag(self, E):
        """v = y * W + x in every pixel of E's state (exact: below 2^24), the costs unchanged.  Tagging the state under test also
        makes its next certified step check that the tags leave the proposal costs unchanged."""
        if self.naive:
            raise ValueError("pixel tags change the image-based energy's cost: v shifts its warp")
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
                mine = np.asarray(planes[i], np.float32)
            else:
                st = O.pm_rng_state(seed, ids[i])
                mine = O.pm_proposal(kind, m, st, pre_l, u, self.MIN, self.MAX)
                if self.tagged and kind in (L.PROP_EXPANSION, L.PROP_RANDOM):
                    nn = O.CvRNG(st).uniform_int(0, u[2] * u[3])
                    sx, sy = u[0] + nn % u[2], u[1] + nn // u[2]
                    T.n_named += 1
                    T.named += int(pre_l[sy, sx, 3] == self.tags[sy, sx] and used[i, 3] == self.tags[sy, sx])
            if kind == L.PROP_RANDOM:
                T.n_random += 1
                assert bits(used[i])[3] == bits(mine)[3] and np.allclose(used[i], mine, rtol=2e-6, atol=1e-6), \
                    f"(P) Random m={m}, cell {ids[i]} unit {u}: device {used[i]!r}, oracle {mine!r}"
                T.random += 1
                T.random_same += int(np.array_equal(bits(used[i]), bits(mine)))
            else:
                T.n_exact += 1
                assert np.array_equal(bits(used[i]), bits(mine)), f"(P) kind {kind}, cell {ids[i]} unit {u}: device {used[i]!r}, oracle {mine!r}"
                T.exact += 1
                T.ransac += int(kind == L.PROP_RANSAC)
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
        if self.naive and self.filter != "GF":
            for i in self.rng.choice(n, min(n, self.q_cells), replace=False):
                x, y, w, h = targets[i]
                ref, scale = self.Or.unary(filters[i], targets[i], used[i], self.mode)
                T.worst_q = max(T.worst_q, FC.compare(q_c[y:y + h, x:x + w], ref, scale, self.filter == "",
                                                      f"(Q) {self.filter!r} cell {ids[i]} plane {used[i]}"))
                T.q_cells += 1
        elif self.naive:
            for i in self.rng.choice(n, min(n, self.q_cells), replace=False):
                x, y, w, h = targets[i]
                ref = self.Or.compute_unary_potential(filters[i], targets[i], used[i], self.mode)
                T.worst_q = max(T.worst_q, assert_costs_close(q_c[y:y + h, x:x + w], ref, f"(Q) cell {ids[i]} plane {used[i]}"))
                T.q_cells += 1
        elif self.filter != "GF":
            if self.fq is None:
                self.fq = (np.empty((self.H, self.W)), np.empty((self.H, self.W)))
            fk = self.C.FILTER_NONE if self.filter == "" else self.C.FILTER_BILATERAL
            ref, scale = self.C.filter_unary_batch(self.mode, filters, targets, used, *self.fq, with_check=True, filter=fk,
                                                   windR=self.windR, sig2=self.sig2)
            T.worst_q = max(T.worst_q, FC.compare(q, ref[inside], scale[inside], self.filter == "", f"(Q) {self.filter!r} step kind {kind} m {m}"))
            T.q_cells += n
        else:
            ref = np.zeros((self.H, self.W), np.float32)
            self.C.unary_batch(self.mode, filters, targets, used, ref, with_check=True)
            r = ref[inside]
            nan = np.isnan(r)
            assert np.array_equal(nan, np.isnan(q)), f"(Q) NaN pattern differs at {int((nan != np.isnan(q)).sum())} pixels"
            T.worst_q = max(T.worst_q, assert_costs_close(q[~nan], r[~nan], f"(Q) step kind {kind} m {m}"))
            T.q_cells += n
        T.t_oracle += time.perf_counter() - t1
        # (I)
        img = dm.zeros((self.H, self.W), fill=np.nan)
        plan.eval_device(dm.ptr(rec), dm.ptr(img), self.W * 4, with_check=True, mode=self.mode, planes_on_device=True)
        E.sync()
        ev = np.array(dm.download(img), np.float32)[inside]
        bad = bits(ev) != bits(q)
        assert not bad.any(), (f"(I) the PatchMatch and unary instantiations differ at {int(bad.sum())} of {bad.size} pixels, up to "
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

    def iteration(self, it, seed, certify=lambda g: True, snap_layer=None):
        """One iteration of the sweep under test; steps of the GroupPlans `certify` selects are certified.  Returns (launches, the
        state at the end of layer snap_layer) (None: not taken)."""
        S, snap, launches = self.S, None, 0
        twin = {(g.layer, g.group): g.plan for g in self.Sq.groups}

        def issue(g, steps):
            for k, kind, m, sd, sync in steps:
                if certify(g):
                    self.certify(g, twin[(g.layer, g.group)], kind, m, sd, k, sync=sync)
                else:
                    g.plan.pm_step(k, kind, m, sd, mode=self.mode, **sync)
        for n, count in enumerate(S.walk(it, seed, issue)):
            launches += count
            li = S.schedule[n][0]
            if li == snap_layer and (n + 1 == len(S.schedule) or S.schedule[n + 1][0] != li):
                snap = self.get(self.E)
        return launches, snap

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


def run_sweep(R, labels, iterations, seed, what="scene", layers=None):
    """The twin uninterrupted, then the sweep under test step by step with every step certified (the initialisation included;
    layers: only the steps of these layers, the others issued one by one uncertified); the final states must be bit-identical.
    The cost-volume energy's states are tagged after the initialisation."""
    tag = not R.naive
    ref = R.twin_reference(labels, seed, (iterations - 1, len(R.S.unit_sizes) - 1), tag=tag)
    R.E.pm_begin(R.mode)
    R.init(labels)
    if tag:
        R.tag(R.E)
    for it in range(iterations):
        R.iteration(it, seed, certify=lambda g: layers is None or g.layer in layers)
    assert_same_state(R.get(R.E), ref, f"{what}: step by step against uninterrupted")
    print(R.T.line(what))
    return R.T
