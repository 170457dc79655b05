"""Scenes for the lean build of the fused kernel: lexp_fused_kernel<10, false, true, kLeanCtas>, the cost-volume PatchMatch-phase
kernel at windR 20 / 21 compiled for three resident CTAs per SM (DESIGN.md 3a).  Shared by tests/test_emu_lean.py and
tests/test_gpu_zz_lean.py.

The lean build differs from the two-CTA build in team A's batch (4 rows instead of 6), in when teams C and E issue their loads
(row r of the next chunk right after row r of this one) and in where the tile geometry is computed.  launch_fused picks it only for
launches of more than 2 x #SM work items whose widest item leaves room for three CTAs; LEXP_LEAN=1 at lexp_create forces it for every
R = 10 cost-volume PatchMatch-phase launch and LEXP_LEAN=0 forbids it, without changing the plans.  So:
  check A: contexts under LEXP_LEAN=1, =0 and unset run the same steps on the same inputs; after every step (designed scenes) or
           every group (sweeps) currentCost, currentLabeling and the recorded planes must be bit-identical;
  check B: pm_step_rig.Rig with both contexts under LEXP_LEAN=1: every step certified -- the update rule bit for bit, the lean
           q against the FP64 oracle, and the lean PatchMatch q against the two-CTA unary instantiation bit for bit.
Every check asserts from lexp_lean_launch_count that the build it means to test ran."""
import numpy as np

from lexp_testlib import bits, make_scene, seeded_labels
from pm_step_rig import Rig, assert_same_state, run_sweep

R10 = 10          # windR 20 and 21: the radius the lean build exists for
OW_MAX = 64       # max_tile_ow(10): the planner's widest column tile
SMEM_PER_SM, SMEM_RESERVED_PER_CTA, LEAN_CTAS, MIN_CTAS = 228 * 1024, 1024, 3, 2


# ---- the planner's arithmetic (lexp_plan_create, fused_smem_bytes, launch_fused's rule), to state and check the geometry -----------
def _sidx(x):
    return x + (x >> 3)


def _srow_stride(vw):
    s = _sidx(vw + 8 + 7) + 1
    return s + ((12 - (s & 7)) & 7)


def fused_smem_bytes(ow, oh, R):
    vw, K, vh = ow + 4 * R, 2 * R + 1, oh + 4 * R
    rows = 2 * 2 * (_srow_stride(vw) + 2 * _srow_stride(vw - 2 * R) + _srow_stride(vw - 4 * R))
    return ((K * vw + 1) // 2 + K * (vw - 2 * R) + rows + 3 * ((vh + 3) // 4) + 3) * 16 + 16


def fits_lean(smem):
    return LEAN_CTAS * (smem + SMEM_RESERVED_PER_CTA) <= SMEM_PER_SM


def plan_rows(targets, R, tile_oh=None, num_sms=132):
    """The segment height lexp_plan_create uses: tile_oh when LEXP_TILE_OH is given, else its search over 24 .. 128."""
    if tile_oh is not None:
        return tile_oh
    slots, best, oh_max = MIN_CTAS * num_sms, 1e300, 128
    for cand in range(24, 129, 4):
        items, max_rows = 0, 0
        for t in targets:
            ncol, nrow = -(-t[2] // OW_MAX), -(-t[3] // cand)
            items += ncol * nrow
            max_rows = max(max_rows, -(-t[3] // nrow))
        cost = -(-items // slots) * (max_rows + 4 * R + 12)
        if cost < best - 1e-9:
            best, oh_max = cost, cand
    return oh_max


def plan_items(filters, targets, R, tile_oh=None, num_sms=132):
    """The work items of lexp_plan_create with what the kernel derives from them: VHs streamed rows of the dependency cone, vReal of
    them inside the filterRect, the cone clipped by the filterRect at the top / bottom, the item's shared memory."""
    oh_max = plan_rows(targets, R, tile_oh, num_sms)
    out = []
    for call, (f, t) in enumerate(zip(filters, targets)):
        ncol, nrow = -(-t[2] // OW_MAX), -(-t[3] // oh_max)
        for rj in range(nrow):
            y0, y1 = t[1] + t[3] * rj // nrow, t[1] + t[3] * (rj + 1) // nrow
            for cj in range(ncol):
                x0, x1 = t[0] + t[2] * cj // ncol, t[0] + t[2] * (cj + 1) // ncol
                ys = max(y0 - 2 * R, f[1])
                VHs = y1 + 2 * R - ys
                vReal = min(VHs, f[1] + f[3] - ys)
                out.append(dict(call=call, ow=x1 - x0, oh=y1 - y0, VHs=VHs, vReal=vReal, top=y0 - 2 * R < f[1], bottom=vReal < VHs,
                                cell_items=ncol * nrow, smem=fused_smem_bytes(x1 - x0, y1 - y0, R)))
    return out


def shipped_rule_is_lean(items, num_sms):
    return fits_lean(max(i["smem"] for i in items)) and len(items) > MIN_CTAS * num_sms


def under_lean(monkeypatch, lean, make):
    """make() with LEXP_LEAN=lean in the environment (None: unset), which lexp_create reads."""
    if lean is None:
        monkeypatch.delenv("LEXP_LEAN", raising=False)
    else:
        monkeypatch.setenv("LEXP_LEAN", str(lean))
    try:
        return make()
    finally:
        monkeypatch.delenv("LEXP_LEAN", raising=False)


def params(windR):
    import localexpstereo_b200 as L
    return L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5)


# ---- designed scenes: chosen cells, chosen steps ----------------------------------------------------------------------------------------
class Designed:
    """Cells (unit = target, filterRect = target +- windR clipped to the image) laid out so that the work items take the shapes the
    lean build's batching and flushing can get wrong.  With LEXP_TILE_OH = 128 every target is one row segment:
      * columns of width 64, 60, 33, 8, 7 and 1 in three bands: at the top of the image (the cone clipped by the filterRect at the
        top), in the middle (unclipped) and at the bottom (clipped at the bottom: the flushing zero rows start at vReal < VHs);
        their heights make VHs (and vReal at the bottom) take every residue mod 4, team A's lean batch;
      * the middle 64-wide column is a 64 x 128 item (77,472 bytes: the shipped rule never runs it lean);
      * a 128-wide target (two 64-wide column tiles of one cell), a 1-row target and a 1 x 1 target (flags & 1).
    Smaller LEXP_TILE_OH cut the tall cells into row segments: multi-tile cells whose items hand the proposal over through CellSync.
    Steps: initialisation from designed planes (PROP_LIST), Expansion, Random, the initialisation's planes again (every target pixel
    ties with its lean q: nothing may change), then planes that are NaN, +-inf, steep or out of range (PROP_LIST)."""

    def __init__(self, windR=20, mode=0, MIN=0.0, MAX=None, tile_oh=128, seed=0):
        import localexpstereo_b200 as L
        self.windR, self.mode, self.tile_oh, self.seed = windR, mode, tile_oh, seed
        self.H, self.W, self.D = 300, 320, 24
        self.MIN, self.MAX = float(MIN), float(self.D - 1 if MAX is None else MAX)
        widths = [64, 60, 33, 8, 7, 1]
        xs = np.concatenate([[0], np.cumsum(widths)])
        top_h, mid_h, bot_h = [61, 62, 63, 64, 62, 63], [128, 125, 126, 127, 128, 126], [64, 61, 62, 63, 61, 62]
        ts = []
        for j, w in enumerate(widths):
            ts.append((int(xs[j]), 0, w, top_h[j]))
            ts.append((int(xs[j]), 100, w, mid_h[j]))
            ts.append((int(xs[j]), self.H - bot_h[j], w, bot_h[j]))
        ts += [(184, 100, 128, 128), (200, 10, 1, 1), (230, 30, 40, 1), (190, 40, 20, 33)]
        self.targets = ts
        self.units = list(ts)
        self.filters = [(max(x - windR, 0), max(y - windR, 0), min(x + w + windR, self.W) - max(x - windR, 0),
                         min(y + h + windR, self.H) - max(y - windR, 0)) for (x, y, w, h) in ts]
        self.ids = np.arange(len(ts), dtype=np.int32)
        self.items = plan_items(self.filters, self.targets, R10, tile_oh)
        n = len(ts)
        rs = np.random.default_rng(seed)
        D = self.D
        cx = np.array([x + w / 2 for (x, _, w, _) in ts], np.float32)
        cy = np.array([y + h / 2 for (_, y, _, h) in ts], np.float32)
        a, b = rs.uniform(-0.08, 0.08, n).astype(np.float32), rs.uniform(-0.08, 0.08, n).astype(np.float32)
        c = (rs.uniform(0.3 * D, 0.7 * D, n) - a * cx - b * cy).astype(np.float32)
        self.init_planes = np.stack([a, b, c, np.arange(n, dtype=np.float32)], 1)
        edge = [(np.nan, 0.0, 5.0, 2.0), (0.0, 0.0, np.inf, 1.0), (0.0, 0.0, -np.inf, 1.0), (np.inf, 0.0, 5.0, 1.0),
                (0.0, 0.0, -50.0, 1.0), (0.0, 0.0, D + 30.0, 1.0), (0.0, 0.0, D - 1.0, 1.0), (0.0, 0.0, 0.0, 1.0)]
        odd = []
        for i in range(n):
            if i % 10 == 8:     # steep: the plane runs through most of the disparity range across the tile, and beyond
                s = np.float32(1.5 * D / max(ts[i][2], ts[i][3], 2))
                odd.append((s, -s, np.float32(D / 2) - s * cx[i] + s * cy[i], 3.0))
            elif i % 10 == 9:
                odd.append(tuple(self.init_planes[i]))
            else:
                odd.append(edge[i % 10 % len(edge)])
        self.edge_planes = np.array(odd, np.float32)
        self.steps = [("init", self.init_planes), (L.PROP_EXPANSION, 0), (L.PROP_RANDOM, 1), ("list", self.init_planes),
                      ("list", self.edge_planes), (L.PROP_RANDOM, 3)]

    def scene(self):
        return make_scene(self.H, self.W, self.D, seed=self.seed)

    def state_geometry(self):
        """What the cells above make of the items; for LEXP_TILE_OH = 128 the full coverage of the docstring."""
        it = self.items
        assert all(i["ow"] <= OW_MAX for i in it)
        assert any(i["cell_items"] > 1 for i in it), "no cell is cut into several work items"
        if self.tile_oh == 128:
            for where in ("top", "mid", "bottom"):
                sel = [i for i in it if (i["top"] if where == "top" else i["bottom"] if where == "bottom" else not (i["top"] or i["bottom"]))]
                key = "vReal" if where == "bottom" else "VHs"
                assert {i[key] % 4 for i in sel} == {0, 1, 2, 3}, (where, sorted({i[key] % 4 for i in sel}))
            assert {i["ow"] for i in it} >= {1, 7, 8, 33, 60, 64}
            big = [i for i in it if i["ow"] == 64 and i["oh"] == 128]
            assert big and all(i["smem"] == 77472 and not fits_lean(i["smem"]) for i in big)
            assert any(i["oh"] == 1 for i in it) and any(i["ow"] == 1 and i["oh"] == 1 for i in it)
        return it

    def issue(self, plan, k, step, d_out, mode, seed):
        """Step k of the scene on `plan`, its planes recorded at d_out."""
        import localexpstereo_b200 as L
        kind, arg = step
        if kind in ("init", "list"):
            plan.pm_step(0, L.PROP_LIST, planes=arg, d_planes_out=d_out, init=kind == "init", mode=mode)
        else:
            plan.pm_step(0, kind, arg, seed + k, d_planes_out=d_out, mode=mode)


def designed_ab(devmem, monkeypatch, sc):
    """Check A on a designed scene: after every step the three contexts' states and recorded planes are bit-identical."""
    import localexpstereo_b200 as L
    monkeypatch.setenv("LEXP_TILE_OH", str(sc.tile_oh))
    items = sc.state_geometry()
    imL, imR, volL, volR = sc.scene()
    ctx = {}
    try:
        for lean in (1, 0, None):
            E = under_lean(monkeypatch, lean, lambda: L.CostVolumeEnergy(imL, imR if sc.mode else None, volL, volR if sc.mode else None,
                                                                         params(sc.windR), sc.MAX, sc.MIN))
            plan = E.make_plan(sc.filters, sc.targets)
            plan.set_units(sc.units, sc.ids)
            assert plan.num_items == len(items), (plan.num_items, len(items))
            E.pm_begin(sc.mode)
            ctx[lean] = (E, plan)
        n = len(sc.targets)
        for k, step in enumerate(sc.steps):
            got = {}
            for lean, (E, plan) in ctx.items():
                E.pm_reset_sync()
                rec = devmem.zeros((n, 4), fill=np.nan)
                sc.issue(plan, k, step, devmem.ptr(rec), sc.mode, 100 * sc.seed + 7)
                E.sync()
                got[lean] = (E.pm_get(sc.mode), np.array(devmem.download(rec), np.float32))
            for lean in (0, None):
                what = f"step {k} ({step[0]}), LEXP_LEAN=1 against LEXP_LEAN={lean}"
                assert_same_state(got[1][0], got[lean][0], what)
                assert np.array_equal(bits(got[1][1]), bits(got[lean][1])), f"{what}: recorded planes differ"
        assert ctx[1][0].lean_launch_count == len(sc.steps), ctx[1][0].lean_launch_count
        assert ctx[0][0].lean_launch_count == 0
        # the shipped rule: these plans are far below 2 x #SM items
        assert ctx[None][0].lean_launch_count == 0
    finally:
        for E, plan in ctx.values():
            plan.close()
            E.close()


def designed_certified(devmem, monkeypatch, sc):
    """Check B on a designed scene: every step of the lean build certified by Rig.certify."""
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import GroupPlan
    monkeypatch.setenv("LEXP_TILE_OH", str(sc.tile_oh))
    sc.state_geometry()
    imL, imR, volL, volR = sc.scene()
    R = under_lean(monkeypatch, 1, lambda: Rig(devmem, imL, imR, volL, volR, sc.windR, [sc.W], [[(L.PROP_EXPANSION, 1)]], sc.mode,
                                               sc.MIN, sc.MAX))
    g = gq = None
    try:
        g, gq = [GroupPlan(0, 0, sc.ids, E.make_plan(sc.filters, sc.targets), 0, sc.units, sc.targets, sc.filters, sc.ids)
                 for E in (R.E, R.Eq)]
        for x in (g, gq):
            x.plan.set_units(sc.units, sc.ids)
        R.E.pm_begin(sc.mode)
        R.Eq.pm_begin(sc.mode)
        for k, (kind, arg) in enumerate(sc.steps):
            R.E.pm_reset_sync()
            if kind in ("init", "list"):
                pre, post, inside, q = R.certify(g, gq.plan, L.PROP_LIST, planes=arg, init=kind == "init")
                if kind == "list" and arg is sc.init_planes:   # the planes the state holds: every target pixel ties with its q
                    assert np.array_equal(bits(post[0]), bits(pre[0])) and np.array_equal(bits(post[1]), bits(pre[1])), \
                        "a tie between the current cost and the lean q changed the state"
                    assert np.isfinite(q).all()
            else:
                R.certify(g, gq.plan, kind, arg, 100 * sc.seed + 7 + k)
        assert R.T.steps == len(sc.steps)
        assert R.E.lean_launch_count == R.T.steps, (R.E.lean_launch_count, R.T.steps)   # the unary launches of (I) are never lean
        assert R.Eq.lean_launch_count > 0
        print(R.T.line(f"lean build, designed cells, windR {sc.windR}, mode {sc.mode}, LEXP_TILE_OH {sc.tile_oh}"))
    finally:
        for x in (g, gq):
            if x is not None:
                x.plan.close()
        R.close()


# ---- sweeps: the LayerManager's cells, several layers, the sweep's own schedule -------------------------------------------------------
class SweepScene:
    """A ragged image (the last unit of every row and column is wider), two layers of windR 20 / 21 cells, Expansion and Random; LEXP_TILE_OH cuts the cells into
    row segments (several work items per cell)."""

    def __init__(self, windR=20, mode=0, MIN=0.0, MAX=None, tile_oh=12, seed=0, H=90, W=106, D=16, units=(24, 52)):
        import localexpstereo_b200 as L
        self.windR, self.mode, self.tile_oh, self.seed, self.H, self.W, self.D = windR, mode, tile_oh, seed, H, W, D
        self.MIN, self.MAX = float(MIN), float(D - 1 if MAX is None else MAX)
        self.units = list(units)
        self.proposers = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)]]

    def scene(self):
        return make_scene(self.H, self.W, self.D, seed=self.seed)

    def check_geometry(self, S):
        for g in S.groups:
            assert g.plan.num_items == len(plan_items(g.filters, g.targets, R10, self.tile_oh)), "the planner replica disagrees"
        assert any(g.plan.num_items > g.plan.num_calls for g in S.groups), "no cell is cut into several work items"
        for lay in S.lm.layers:
            assert len({u[2] for u in lay.unitRegions}) > 1 and len({u[3] for u in lay.unitRegions}) > 1, "the image should be ragged"


def sweep_ab(devmem, monkeypatch, sc, iterations=1):
    """Check A on a sweep: the initialisation and `iterations` pm iterations on three contexts, compared at the end of every group."""
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import PMSweep
    monkeypatch.setenv("LEXP_TILE_OH", str(sc.tile_oh))
    imL, imR, volL, volR = sc.scene()
    ctx = {}
    try:
        for lean in (1, 0, None):
            E = under_lean(monkeypatch, lean, lambda: L.CostVolumeEnergy(imL, imR if sc.mode else None, volL, volR if sc.mode else None,
                                                                         params(sc.windR), sc.MAX, sc.MIN))
            ctx[lean] = (E, PMSweep(E, unit_sizes=sc.units, proposers=sc.proposers, mode=sc.mode))
        S1 = ctx[1][1]
        sc.check_geometry(S1)
        labels = seeded_labels(S1, 11 + sc.seed)
        launches = compare_walks(devmem, {k: v[1] for k, v in ctx.items()}, labels, iterations, 500 + sc.seed)
        assert ctx[1][0].lean_launch_count == sum(launches.values()) > 0
        assert ctx[0][0].lean_launch_count == 0 and ctx[None][0].lean_launch_count == 0
    finally:
        for E, S in ctx.values():
            S.close()
            E.close()


def compare_walks(devmem, sweeps, labels, iterations, seed, on_layer_end=None):
    """The initialisation and pm iterations 0 .. iterations - 1 of every sweep in `sweeps` ({LEXP_LEAN: PMSweep}, key 1 required), one
    group at a time on all of them; after every group the states and the recorded planes must equal those of sweeps[1] bit for bit.
    on_layer_end(it, layer) is called at the end of every layer (it None: the initialisation).  Returns {(it, layer): launches}."""
    import localexpstereo_b200 as L
    keys = list(sweeps)
    mode = sweeps[1].mode
    launches = {}

    def recorder(key, rec):
        def issue(g, steps):
            rec.clear()
            for k, kind, m, sd, sync in steps:
                buf = devmem.zeros((g.plan.num_calls, 4), fill=np.nan)
                rec.append(buf)
                if kind == L.PROP_LIST:
                    g.plan.pm_step(k, kind, planes=labels, d_planes_out=devmem.ptr(buf), init=True, mode=mode, **sync)
                else:
                    g.plan.pm_step(k, kind, m, sd, d_planes_out=devmem.ptr(buf), mode=mode, **sync)
        return issue

    for S in sweeps.values():
        S.begin()
    for it in [None] + list(range(iterations)):
        recs = {k: [] for k in keys}
        walks = [sweeps[k].walk(it, seed, recorder(k, recs[k])) for k in keys]
        sched = [(0, 0)] if it is None else [(li, gi) for (li, gi, _, _) in sweeps[1].schedule]
        for n, counts in enumerate(zip(*walks)):
            li, gi = sched[n]
            launches[(it, li)] = launches.get((it, li), 0) + counts[0]
            states = {k: sweeps[k].get() for k in keys}
            planes = {k: [np.array(devmem.download(b), np.float32) for b in recs[k]] for k in keys}
            for k in keys:
                if k == 1:
                    continue
                what = f"{'initialisation' if it is None else f'iteration {it}'}, layer {li}, group {gi}: LEXP_LEAN=1 against LEXP_LEAN={k}"
                assert_same_state(states[1], states[k], what)
                assert len(planes[1]) == len(planes[k]) and all(np.array_equal(bits(a), bits(b)) for a, b in zip(planes[1], planes[k])), \
                    f"{what}: recorded planes differ"
            if on_layer_end and (n + 1 == len(sched) or sched[n + 1][0] != li):
                on_layer_end(it, li)
        for w in walks:   # run the walks to their end: the epoch base advances there
            for _ in w:
                raise AssertionError("the walks have different lengths")
    return launches


def sweep_certified(devmem, monkeypatch, sc, iterations=1):
    """Check B on a sweep: pm_step_rig.run_sweep with both contexts under LEXP_LEAN=1."""
    monkeypatch.setenv("LEXP_TILE_OH", str(sc.tile_oh))
    imL, imR, volL, volR = sc.scene()
    R = under_lean(monkeypatch, 1, lambda: Rig(devmem, imL, imR, volL, volR, sc.windR, sc.units, sc.proposers, sc.mode, sc.MIN, sc.MAX))
    try:
        sc.check_geometry(R.S)
        T = run_sweep(R, seeded_labels(R.S, 11 + sc.seed), iterations, 500 + sc.seed,
                      what=f"lean build, sweep, windR {sc.windR}, mode {sc.mode}, LEXP_TILE_OH {sc.tile_oh}")
        assert R.E.lean_launch_count == T.steps > 0, (R.E.lean_launch_count, T.steps)
        assert R.Eq.lean_launch_count > 0
    finally:
        R.close()
