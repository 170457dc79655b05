"""The PatchMatch phase of the image-based energy (NaiveStereoEnergy, `-mode MiddV2`) on the device, step by step against the
oracle's update of the SAME state: shared by tests/test_gpu_zz_naive_pm.py and tests/test_emu_naive_pm.py.

Every step starts from the device's own pre-step state (pm_get) and is certified without a budget (NaiveRig.certify):
  (P) proposal: the oracle's proposer on the device's pre-step labeling, with the launch's random stream, gives the plane the step
      recorded -- bit for bit for lists, ExpansionProposer and RansacProposer; RandomProposer within 2e-6 relative / 1e-6 absolute
      (CUDA's FP64 sin / cos against glibc's), its fourth component bit for bit;
  (U) update: nothing outside the group's targetRects changes; inside, post = (pre_cost > q) ? (q, plane) : pre bit for bit, or
      (q, plane) unconditionally for an initialisation.  q is the PatchMatch instantiation's own proposal cost: the recorded planes
      run as an initialisation (pm_mode 2) on a twin context with the same inputs;
  (I) q equals the unary instantiation's cost of the same planes (Plan.eval_device: image output, with the check) bit for bit;
  (Q) q against the numpy oracle of the energy on a sample of the step's cells: 1e-4 relative and the exact COST_FOR_INVALID mask.
Pixel tags (tests/test_gpu_zz_pm_steps.py) cannot name source pixels here: v shifts this energy's warp, so it changes the cost.
A whole-run replay would drift at the exact FP32 ties of the truncated image cost (tests/test_gpu_zz_gc.py explains them); a
per-step certification does not."""
import time

import numpy as np

import ransac_oracle as RO
from oracle import lexp_oracle as O
from lexp_testlib import assert_costs_close, bits, seeded_labels

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


class Tally:
    def __init__(self):
        self.steps = self.exact = self.n_exact = self.random = self.n_random = self.q_cells = 0
        self.worst_q = 0.0
        self.t_step = 0.0

    def line(self, what):
        return (f"{what}: {self.steps} steps certified; proposals bit-identical {self.exact} of {self.n_exact} (list / Expansion / RANSAC), "
                f"Random within tolerance {self.random} of {self.n_random}; (Q) {self.q_cells} cells, worst err {self.worst_q:.2e}; "
                f"{self.t_step:.1f} s")


class NaiveRig:
    """The context under test E and its twin Eq on the same images, a PMSweep on each, and the numpy oracle of the energy."""

    def __init__(self, devmem, imL, imR, D, windR, units, proposers, mode=0, q_cells=4, seed=0):
        import localexpstereo_b200 as L
        from localexpstereo_b200.sweep import PMSweep
        self.L, self.dm, self.mode, self.q_cells = L, devmem, mode, q_cells
        prm = middv2_params(windR)
        self.MAX = float(D - 1)
        self.E, self.Eq = [L.NaiveStereoEnergy(imL, imR, prm, self.MAX) for _ in range(2)]
        self.H, self.W = self.E.height, self.E.width
        self.S, self.Sq = [PMSweep(E, unit_sizes=units, proposers=proposers, mode=mode) for E in (self.E, self.Eq)]
        self.Or = O.NaiveStereoEnergyOracle(imL, imR, windR, 1e-4, prm.th_col, prm.th_grad, prm.alpha, self.MAX)
        self.rng = np.random.default_rng(seed)
        self.owner = {}
        self.T = Tally()

    def close(self):
        for S in (self.S, self.Sq):
            S.close()
        for E in (self.E, self.Eq):
            E.close()

    def owner_of(self, targets):
        key = tuple(map(tuple, targets))
        if key not in self.owner:
            o = np.full((self.H, self.W), -1, np.int64)
            for i, (x, y, w, h) in enumerate(targets):
                assert (o[y:y + h, x:x + w] == -1).all(), "targetRects of one step overlap"
                o[y:y + h, x:x + w] = i
            self.owner[key] = o
        return self.owner[key]

    def twin_q(self, qplan, d_planes):
        """The PatchMatch instantiation's cost of the planes in every target pixel: an initialisation step on the twin."""
        self.Eq.pm_reset_sync()
        qplan.pm_step(0, self.L.PROP_LIST, planes=d_planes, planes_on_device=True, init=True, mode=self.mode)
        self.Eq.sync()
        return self.Eq.pm_get(self.mode)

    def certify(self, g, qplan, kind, m=0, seed=0, step_index=0, init=False, planes=None, sync=None):
        L, E, dm, T = self.L, self.E, self.dm, self.T
        t0 = time.perf_counter()
        plan, units, targets, filters, ids = g.plan, g.units, g.targets, g.filters, g.ids
        n = plan.num_calls
        assert len(units) == n and (kind == L.PROP_LIST) == (planes is not None)
        E.sync()
        pre_c, pre_l = E.pm_get(self.mode)
        rec = dm.zeros((n, 4), fill=np.nan)
        plan.pm_step(step_index, kind, m, seed, planes=planes, d_planes_out=dm.ptr(rec), init=init, mode=self.mode, **(sync or {}))
        E.sync()
        post_c, post_l = E.pm_get(self.mode)
        used = np.array(dm.download(rec), np.float32)
        # (P)
        for i, u in enumerate(units):
            if kind == L.PROP_LIST:
                mine = np.asarray(planes[i], np.float32)
            else:
                mine = RO.proposal(kind, m, O.pm_rng_state(seed, ids[i]), pre_l, u, 0.0, self.MAX)
            if kind == L.PROP_RANDOM:
                T.n_random += 1
                assert bits(used[i])[3] == bits(mine)[3] and np.allclose(used[i], mine, rtol=2e-6, atol=1e-6), \
                    f"(P) Random m={m}, cell {ids[i]} unit {u}: device {used[i]!r}, oracle {mine!r}"
                T.random += 1
            else:
                T.n_exact += 1
                assert np.array_equal(bits(used[i]), bits(mine)), f"(P) kind {kind}, cell {ids[i]} unit {u}: device {used[i]!r}, oracle {mine!r}"
                T.exact += 1
        # q: the PatchMatch instantiation, on the twin
        q_c, q_l = self.twin_q(qplan, dm.ptr(rec))
        own = self.owner_of(targets)
        inside = own >= 0
        plane_px = used[own[inside]]
        q = q_c[inside]
        assert np.array_equal(bits(q_l[inside]), bits(plane_px)), "the twin's initialisation did not write the recorded planes"
        # (U)
        pc, pl = pre_c[inside], pre_l[inside]
        upd = np.ones(q.shape, bool) if init else pc > q
        assert np.array_equal(bits(post_c[inside]), bits(np.where(upd, q, pc))), \
            f"(U) cost: {int((bits(post_c[inside]) != bits(np.where(upd, q, pc))).sum())} target pixels differ from the rule"
        assert np.array_equal(bits(post_l[inside]), bits(np.where(upd[:, None], plane_px, pl))), "(U) label differs from the rule"
        assert np.array_equal(bits(post_c[~inside]), bits(pre_c[~inside])) and np.array_equal(bits(post_l[~inside]), bits(pre_l[~inside])), \
            "(U) a pixel outside the step's targetRects changed"
        # (I)
        img = dm.zeros((self.H, self.W), fill=np.nan)
        plan.eval_device(dm.ptr(rec), dm.ptr(img), self.W * 4, with_check=True, mode=self.mode, planes_on_device=True)
        E.sync()
        ev = np.array(dm.download(img), np.float32)[inside]
        bad = bits(ev) != bits(q)
        assert not bad.any(), f"(I) the PatchMatch and unary instantiations differ at {int(bad.sum())} of {bad.size} pixels"
        # (Q) on a sample of the cells
        for i in self.rng.choice(n, min(n, self.q_cells), replace=False):
            x, y, w, h = targets[i]
            ref = self.Or.compute_unary_potential(filters[i], targets[i], used[i], self.mode)
            T.worst_q = max(T.worst_q, assert_costs_close(q_c[y:y + h, x:x + w], ref, f"(Q) cell {ids[i]} plane {used[i]}"))
            T.q_cells += 1
        T.steps += 1
        T.t_step += time.perf_counter() - t0

    # ---- the sweep's own walk, one step at a time ---------------------------------------------------------------------------------------
    def init(self, labels):
        def issue(g, steps):
            ((k, kind, _, _, sync),) = steps
            self.certify(g, self.Sq.init_plan, kind, planes=np.asarray(labels, np.float32), init=True, sync=sync)
        for _ in self.S.walk(None, 0, issue):
            pass

    def iteration(self, it, seed, certify=lambda g: True):
        twin = {(g.layer, g.group): g.plan for g in self.Sq.groups}

        def issue(g, steps):
            for k, kind, m, sd, sync in steps:
                if certify(g):
                    self.certify(g, twin[(g.layer, g.group)], kind, m, sd, k, sync=sync)
                else:
                    g.plan.pm_step(k, kind, m, sd, mode=self.mode, **sync)
        return sum(self.S.walk(it, seed, issue))


def run_certified(R, labels, iterations, seed, what):
    """The initialisation (a LEXP_PM_INIT step of the PatchMatch-phase kernel) and `iterations` pm iterations, every step certified;
    the final state must equal the twin's uninterrupted sweep (PMSweep.init / iteration) bit for bit."""
    R.Sq.begin()
    R.Sq.init(labels)
    for it in range(iterations):
        R.Sq.iteration(it, seed)
    ref = R.Sq.get()
    R.S.begin()
    R.init(labels)
    for it in range(iterations):
        R.iteration(it, seed)
    got = R.S.get()
    assert np.array_equal(bits(got[0]), bits(ref[0])) and np.array_equal(bits(got[1]), bits(ref[1])), \
        f"{what}: step by step against uninterrupted"
    print(R.T.line(what))
    return R.T


# ---- scenes --------------------------------------------------------------------------------------------------------------------------------
def reference_lists(n_layers):
    from localexpstereo_b200.sweep import V3_PROPOSERS_REFERENCE
    return V3_PROPOSERS_REFERENCE[:n_layers]


def scene_cones(devmem, mode, H=None, W=None, units=None, iterations=2, seed=3):
    """The cones crop at windR 20 with the reference's proposer lists (RANSAC included) and MiddV2's layers."""
    imL, imR = cones(H, W)
    units = units or MIDDV2_UNITS
    R = NaiveRig(devmem, imL, imR, 64, 20, units, reference_lists(len(units)), mode, seed=seed)
    try:
        T = run_certified(R, seeded_labels(R.S, 40 + seed), iterations, 500 + seed, f"cones crop {R.H} x {R.W}, windR 20, mode {mode}")
        assert T.n_exact > 50 and T.n_random > 50
        return T
    finally:
        R.close()


def scene_generic_radius(devmem, mode=0, H=61, W=83, iterations=2):
    """windR 12: the generic-radius instantiation <0, true, true>, on a ragged synthetic pair."""
    import localexpstereo_b200 as L
    imL, imR = O.synthetic_image(H, W, 52), O.synthetic_image(H, W, 53)
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANSAC, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]]
    R = NaiveRig(devmem, imL, imR, 24, 12, [7, 19], props, mode, seed=1)
    try:
        T = run_certified(R, seeded_labels(R.S, 11), iterations, 77, f"synthetic {H} x {W}, windR 12, mode {mode}")
        assert T.n_exact > 50 and T.n_random > 50
        return T
    finally:
        R.close()


def scene_vertical_offset(devmem, mode=1, H=72, W=96):
    """Planes with v != 0 (the proposers copy v): the warp shifted vertically, on the cones crop."""
    import localexpstereo_b200 as L
    imL, imR = cones(H, W)
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]]
    R = NaiveRig(devmem, imL, imR, 32, 20, [5, 15], props, mode, seed=2)
    try:
        labels = with_v(seeded_labels(R.S, 9), 9)
        T = run_certified(R, labels, 1, 31, f"v != 0, cones crop {H} x {W}, mode {mode}")
        lab = R.S.get()[1]
        assert (lab[..., 3] != 0).all()
        return T
    finally:
        R.close()
