"""The parity protocols of the device sweeps, shared by the PatchMatch, graph-cut and RANSAC tests.

Replay (run_pm_replay / run_gc_replay): the device sweep records the plane (and, for a graph-cut step, the minimum-cut energy) every
(cell, step) evaluated; the oracle starts from the same initialisation and replays that fixed plane sequence step by step, walking
the sweep's own steps and cell geometry.  At every step the oracle's own proposer, run on the oracle's state with the launch's random
stream, is compared with the recorded plane; check_pm_result / check_gc_result then compare the final states.

Moves (certify_gc_step): one graph-cut step of a plan against the exact minimum cut of the same graph, move by move (the criteria are
stated in tests/test_gpu_zz_gc_moves.py)."""
import math
import time

import numpy as np

from oracle import c_oracle
from oracle import lexp_oracle as O
from lexp_testlib import ABS_FLOOR, REL_TOL, bits, energy_and_oracle, make_scene, seeded_labels

SMOOTH = dict(lam=0.6, omega=10.0, th_smooth=1.0, epsilon=0.01)


# ---- replay ----------------------------------------------------------------------------------------------------------------------------
def recording(devmem, S, iteration, seed, gc=False):
    """Buffers for one iteration's planes_out (and flows_out): {(layer, group): [steps][n][4] floats}, {(layer, group): [steps][n] doubles}."""
    planes, flows = {}, {}
    for g in S.groups:
        n_steps = len(S.group_steps(g.layer, g.group, iteration, seed))
        planes[(g.layer, g.group)] = devmem.zeros((n_steps, g.plan.num_calls, 4))
        if gc:
            flows[(g.layer, g.group)] = devmem.zeros((n_steps, g.plan.num_calls, 2))
    return planes, flows


def pointers(devmem, bufs):
    return {k: devmem.ptr(v) for k, v in bufs.items()}


def oracle_init(Or, S, labels):
    """The oracle's state after initCurrentFast with `labels`, on the sweep's initialisation geometry."""
    H, W = S.energy.height, S.energy.width
    cost, lab = np.full((H, W), np.inf, np.float32), np.zeros((H, W, 4), np.float32)
    g = S.init_group
    O.pm_step(Or, g.units, g.targets, g.filters, 0, 0, 0, None, cost, lab, planes=labels, init=True, mode=S.mode)
    return cost, lab


def oracle_replay(Or, S, cost_o, lab_o, passes, planes, flows=None, smooth=None, coeff=None):
    """The oracle half: from the state (cost_o, lab_o), which it updates in place, the oracle replays the iterations
    passes = [(gc, iteration, seed)] of the sweep S with the planes the device recorded, planes[p][(layer, group)] = [steps][n][4]
    (graph-cut passes: the minimum-cut energies flows[p][(layer, group)] = [steps][n], compared with the oracle's).  Returns the
    oracle's state and the counts check_pm_result / check_gc_result read."""
    lo, hi = S.energy.MIN_DISPARITY, S.energy.MAX_DISPARITY
    n_prop = n_same = n_close = n_moves = 0
    worst_flow = 0.0
    for p, (gc, it, seed) in enumerate(passes):
        for g in S.groups:
            for k, kind, m, sd in S.group_steps(g.layer, g.group, it, seed):
                dev_planes = planes[p][(g.layer, g.group)][k]
                for i, u in enumerate(g.units):   # the oracle's proposer on the oracle's state
                    mine = O.pm_proposal(kind, m, O.pm_rng_state(sd, g.ids[i]), lab_o, u, lo, hi)
                    n_prop += 1
                    n_same += int(np.array_equal(mine, dev_planes[i]))
                    n_close += int(np.allclose(mine, dev_planes[i], rtol=2e-6, atol=1e-6))
                if not gc:
                    O.pm_step(Or, g.units, g.targets, g.filters, 0, 0, 0, None, cost_o, lab_o, planes=dev_planes, mode=S.mode)
                    continue
                _, fo = O.gc_step(Or, g.units, g.targets, g.filters, 0, 0, 0, None, cost_o, lab_o, coeff, smooth["lam"], smooth["th_smooth"],
                                  planes=dev_planes, mode=S.mode)
                df = flows[p][(g.layer, g.group)][k]
                worst_flow = max(worst_flow, float((np.abs(df - fo) / np.maximum(np.abs(fo), 1e-3)).max()))
                n_moves += len(g.units)
    return dict(cost_o=cost_o, lab_o=lab_o, n_prop=n_prop, n_same=n_same, n_close=n_close, n_moves=n_moves, worst_flow=worst_flow)


def replay(devmem, S, Or, seed, pm_iterations, gc_iterations=0, smooth=None, coeff=None):
    """The whole protocol on the sweep S: begin, initialisation with seeded_labels(S, seed), pm iterations 0 .. pm_iterations - 1
    (seed), then graph-cut iterations 0 .. gc_iterations - 1 (seed + 1: both loops of FastGCStereo::run restart `iteration` at 0,
    FastGCStereo.h:143,171), recorded; then the oracle's replay.  Graph-cut passes: also the total energy of both final states."""
    E = S.energy
    passes = [(False, it, seed) for it in range(pm_iterations)] + [(True, it, seed + 1) for it in range(gc_iterations)]
    labels = seeded_labels(S, seed)
    S.begin()
    S.init(labels)
    rec = []
    for gc, it, sd in passes:
        planes, flows = recording(devmem, S, it, sd, gc)
        if gc:
            S.gc_iteration(it, sd, planes_out=pointers(devmem, planes), flows_out=pointers(devmem, flows))
        else:
            S.iteration(it, sd, planes_out=pointers(devmem, planes))
        rec.append((planes, flows))
    E.sync()
    cost_d, lab_d = S.get()
    planes = [{k: devmem.download(v) for k, v in p.items()} for p, _ in rec]
    flows = [{k: np.ascontiguousarray(devmem.download(v)).view(np.float64)[..., 0] for k, v in f.items()} for _, f in rec]
    cost_o, lab_o = oracle_init(Or, S, labels)
    r = dict(oracle_replay(Or, S, cost_o, lab_o, passes, planes, flows, smooth, coeff), cost_d=cost_d, lab_d=lab_d)
    if gc_iterations:
        lam, th = smooth["lam"], smooth["th_smooth"]
        r["e_d"] = float(cost_d.astype(np.float64).sum()) + O.smoothness_cost(lab_d, coeff, lam, th)
        r["e_o"] = float(r["cost_o"].astype(np.float64).sum()) + O.smoothness_cost(r["lab_o"], coeff, lam, th)
    return r


def run_pm_replay(devmem, H, W, D, windR, units, proposers, iterations=1, seed=1234, scene=None, mode=0):
    """`iterations` pm iterations of a PMSweep over view `mode` of a synthetic (or the given) scene, replayed by the oracle."""
    from localexpstereo_b200.sweep import PMSweep
    E, Or = energy_and_oracle(scene if scene is not None else make_scene(H, W, D), D, windR, mode)
    S = PMSweep(E, unit_sizes=units, proposers=proposers, mode=mode)
    try:
        return replay(devmem, S, Or, seed, iterations)
    finally:
        S.close()
        E.close()


def run_gc_replay(devmem, H, W, D, windR, units, proposers, pm_iterations=1, gc_iterations=1, seed=1234, mode=0, smooth=SMOOTH, scene=None,
                  naive=False):
    """pm iterations, then graph-cut iterations of a GCSweep, replayed by the oracle.  naive: the image-based energy of -mode MiddV2
    (no cost volume, no device PatchMatch phase: graph-cut iterations only)."""
    from localexpstereo_b200.sweep import GCSweep
    assert not (naive and pm_iterations)
    scene = scene if scene is not None else make_scene(H, W, D)
    E, Or = energy_and_oracle(scene, D, windR, mode, naive, **(dict(lambda_=smooth["lam"]) if naive else {}))
    S = GCSweep(E, unit_sizes=units, proposers=proposers, mode=mode, **smooth)
    coeff = O.smoothness_coeff(scene[1] if mode else scene[0], smooth["omega"], smooth["epsilon"])
    try:
        return replay(devmem, S, Or, seed, pm_iterations, gc_iterations, smooth, coeff)
    finally:
        S.close()
        E.close()


def check_pm_result(r):
    cd, co, ld, lo = r["cost_d"], r["cost_o"], r["lab_d"], r["lab_o"]
    assert np.isfinite(co).all() == np.isfinite(cd).all()
    inv = co == O.COST_FOR_INVALID
    assert np.array_equal(inv, cd == O.COST_FOR_INVALID)
    err = np.abs(cd.astype(np.float64) - co) / (REL_TOL * np.maximum(np.abs(co), ABS_FLOOR))
    assert err[~inv].max() <= 1.0, f"final cost: max err/tol {err[~inv].max():.3f}"
    diff = (ld != lo).any(axis=2)
    # a differing label is only acceptable where the two competing costs agree within the tolerance (checked above for the winner:
    # the costs are within 1e-4 of each other at such pixels) and must be rare
    assert diff.mean() < 2e-4, f"{diff.sum()} of {diff.size} labels differ"
    assert r["n_close"] == r["n_prop"], (r["n_close"], r["n_prop"])          # every proposal reproduced (FP64 sin/cos: 1e-6)
    assert r["n_same"] >= 0.98 * r["n_prop"], (r["n_same"], r["n_prop"])      # and almost all of them bit for bit
    print(f"pm replay: {r['n_prop']} proposals ({r['n_same']} bit-identical), final cost max err/tol {err[~inv].max():.3f}, "
          f"{int(diff.sum())} of {diff.size} labels differ")


def check_gc_result(r, max_label_fraction=2e-3):
    cd, co, ld, lo = r["cost_d"], r["cost_o"], r["lab_d"], r["lab_o"]
    diff = (ld != lo).any(axis=2)
    same = ~diff
    inv = co == O.COST_FOR_INVALID
    assert np.array_equal(inv[same], (cd == O.COST_FOR_INVALID)[same])
    err = np.abs(cd.astype(np.float64) - co) / (REL_TOL * np.maximum(np.abs(co), ABS_FLOOR))
    sel = same & ~inv
    assert err[sel].max() <= 1.0, f"final cost: max err/tol {err[sel].max():.3f}"
    assert r["n_moves"] > 0 and r["worst_flow"] <= 1e-5, f"minimum-cut energy of a move: rel err {r['worst_flow']:.2e}"
    assert diff.mean() <= max_label_fraction, f"{diff.sum()} of {diff.size} labels differ"
    assert abs(r["e_d"] - r["e_o"]) <= 1e-5 * abs(r["e_o"]), (r["e_d"], r["e_o"])
    assert r["n_close"] >= r["n_prop"] - 2 * int(diff.sum()), (r["n_close"], r["n_prop"])   # a differing label can be drawn as a proposal source
    print(f"gc replay: {r['n_moves']} moves, min-cut energy max rel err {r['worst_flow']:.1e}, final cost max err/tol {err[sel].max():.3f}, "
          f"{int(diff.sum())} of {diff.size} labels differ, energy {r['e_d']:.6f} vs {r['e_o']:.6f}")


# ---- graph-cut moves against the exact minimum cut ---------------------------------------------------------------------------------
U = 2.0 ** -53
ARCS = ((1, 0), (0, 1), (-1, 1), (1, 1))      # the forward arcs GE, EG, LG, GG: cap[0..3] of oracle.expansion_graph
REPORT = dict(worst=0.0, moves=0, ties=0, phase_nodes=0)


def cut_value(tr, cap, mask):
    """Value of the cut `mask` (True = SOURCE side) of the graph (tr, cap), the float32 capacities summed exactly in double: a node outside
    the mask pays its source arc max(tr, 0), a node inside pays its sink arc max(-tr, 0), an arc from inside to outside pays its capacity."""
    terms = [np.where(mask, np.maximum(-tr, 0), np.maximum(tr, 0)).astype(np.float64).ravel()]
    h, w = mask.shape
    for fi, (dx, dy) in enumerate(ARCS):
        xs, xd = slice(max(-dx, 0), w - max(dx, 0)), slice(max(dx, 0), w + min(dx, 0))
        cut = mask[:h - dy, xs] & ~mask[dy:, xd]
        terms.append(cap[fi][:h - dy, xs][cut].astype(np.float64))
    return math.fsum(np.concatenate(terms))


def assert_non_adjacent(regions):
    """The moves of one step read their neighbours' labels: the cells must not touch, diagonals included."""
    for i, (x, y, w, h) in enumerate(regions):
        for (x2, y2, w2, h2) in regions[i + 1:]:
            assert x2 > x + w or x > x2 + w2 or y2 > y + h or y > y2 + h2, ((x, y, w, h), (x2, y2, w2, h2))


def proposal_costs(E, plan, planes, mode, devmem):
    """The image lexp_plan_gc_step evaluates its proposals into: the same plan's unary launch with image output and the validity check."""
    d = devmem.zeros((E.height, E.width), fill=np.nan)
    plan.eval_device(np.asarray(planes, np.float32), devmem.ptr(d), E.width * 4, with_check=True, mode=mode)
    E.sync()
    return np.array(devmem.download(d), np.float32)


def certify_gc_step(E, plan, regions, mode, lam, th, devmem, planes=None, kind=0, m=0, seed=0, exact=False, ties_ok=False, coeff=None,
                    state=None):
    """One proposal step of `plan` (Plan.gc_step: PROP_LIST with `planes`, or a device proposer) checked move by move, (a) to (d) of
    tests/test_gpu_zz_gc_moves.py.  Returns one record per cell.
    Tolerance of (b) to (d): 1e-6 * max(mf, 1e-3).  (b) also allows the double rounding of konst (the device sums it per thread and per
    block, the oracle per node and pairwise): 2 N u * (|konst| + mf + 8 N lam th) bounds any summation order of N terms whose
    absolute values add up to at most that (a node's konst terms are >= -4 lam th).  exact: no tolerance at all.
    coeff: the view's coefficient maps (E.smooth_coeff(mode)) when the caller already holds them (downloaded on every call otherwise).
    state: a dict carrying the device state from one step to the next: its "cost" / "label" are taken as the pre-move state when
    present (downloaded otherwise), and the post-move state is stored there, with "step_s" (wall time of the step up to its
    synchronisation) and "phase" (whether the phase kernels ran it: a one-CTA step is the unary launches of the plan plus at most a
    proposal launch and the move kernel, a phase step issues at least one launch per phase)."""
    import localexpstereo_b200 as L
    H, W = E.height, E.width
    n = len(regions)
    assert_non_adjacent(regions)
    assert (kind == L.PROP_LIST) == (planes is not None)
    if state is not None and "cost" in state:
        pre_c, pre_l = state["cost"], state["label"]
    else:
        pre_c, pre_l = E.pm_get(mode)
    if coeff is None:
        coeff = E.smooth_coeff(mode)
    d_pl, d_fl = devmem.zeros((n, 4)), devmem.zeros((n, 2))
    E.sync()
    n0, t0 = E.launch_count, time.perf_counter()
    plan.gc_step(kind, m, seed, planes=planes, d_planes_out=devmem.ptr(d_pl), d_flows_out=devmem.ptr(d_fl), mode=mode)
    E.sync()
    step_s, n_step = time.perf_counter() - t0, E.launch_count - n0
    post_c, post_l = E.pm_get(mode)
    used = np.array(devmem.download(d_pl), np.float32)
    flows = np.ascontiguousarray(devmem.download(d_fl)).view(np.float64)[:, 0].copy()
    if planes is not None:
        assert np.array_equal(bits(used), bits(np.reshape(planes, (n, 4))))
    n0 = E.launch_count
    q_img = proposal_costs(E, plan, used, mode, devmem)
    if state is not None:
        state.update(cost=post_c, label=post_l, step_s=step_s, phase=n_step - (E.launch_count - n0) > 2)
    inside = np.zeros((H, W), bool)
    cells = []
    for i, reg in enumerate(regions):
        x, y, w, h = (int(v) for v in reg)
        sl = np.s_[y:y + h, x:x + w]
        inside[sl] = True
        q, l1, N = q_img[sl], used[i], w * h
        tr, konst, cap = O.expansion_graph(pre_c, pre_l, q, l1, (x, y, w, h), coeff, lam, th)
        mask_o, mf_o = c_oracle.grid_mincut(tr, cap)
        old = (bits(post_c[sl]) == bits(pre_c[sl])) & (bits(post_l[sl]) == bits(pre_l[sl])).all(axis=2)
        new = (bits(post_c[sl]) == bits(q)) & (bits(post_l[sl]) == bits(l1)).all(axis=2)
        bad = ~(old | new)
        assert not bad.any(), f"(a) cell {(x, y, w, h)}: {int(bad.sum())} pixels hold neither their pre-move state nor the proposal, e.g. {np.argwhere(bad)[0]}"
        either = old & new      # the pre-move state is the proposal already: an isolated node with tr = 0, either side of the cut
        mask_d = new
        v_d, v_o = cut_value(tr, cap, mask_d), cut_value(tr, cap, mask_o)
        tol = 0.0 if exact else 1e-6 * max(mf_o, 1e-3)
        slack = 0.0 if exact else 2 * N * U * (abs(konst) + abs(mf_o) + 8 * N * lam * th)
        err = abs((flows[i] - konst) - v_d)
        diff = (mask_d != mask_o) & ~either
        msg = (f"cell {(x, y, w, h)} ({N} nodes): device flow {flows[i]!r}, konst {konst!r}, oracle max flow {mf_o!r}, cut value of the "
               f"device's mask {v_d!r}, of the oracle's {v_o!r}, {int(diff.sum())} nodes on different sides")
        assert err <= tol + slack, "(b) " + msg
        assert abs(v_d - v_o) <= tol, "(c) " + msg
        assert abs(mf_o - v_o) <= tol + (0.0 if exact else 1e-7 * max(mf_o, 1e-3)), "oracle: " + msg
        assert ties_ok or not diff.any(), "(d) " + msg
        REPORT["worst"] = max(REPORT["worst"], err / max(mf_o, 1e-3))
        REPORT["moves"] += 1
        REPORT["ties"] += int(diff.sum())
        cells.append(dict(region=(x, y, w, h), konst=konst, mf=mf_o, flow=float(flows[i]), mask=mask_d, q=q, ties=int(diff.sum()),
                          err=err / max(mf_o, 1e-3), slack=slack))
    out = ~inside
    assert np.array_equal(bits(post_c[out]), bits(pre_c[out])) and np.array_equal(bits(post_l[out]), bits(pre_l[out])), \
        "(a) a pixel outside the step's cells changed"
    return cells
