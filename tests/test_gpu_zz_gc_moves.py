"""Every graph-cut move of the device against the exact minimum cut of the SAME graph.

The oracle gets the device's own inputs: the pre-move state (pm_get), the device's coefficient maps (smooth_coeff) and the device's proposal
costs (the plan's own unary launch with image output and the validity check, which is what lexp_plan_gc_step writes into its internal
image).  oracle.expansion_graph then builds the graph lexp_gc.cuh builds, bit for bit (same add_tweights order, bit-identical pair terms),
and only the solver is left to compare.  Per move (lexp_replay.certify_gc_step):
  (a) every pixel of a cell holds its pre-move (cost, label) or (proposal cost, proposal), bit for bit; nothing outside the cells changes;
  (b) duality: the device's flow minus BK's constant `konst` equals the value of the device's own cut; a flow and a cut of equal value are
      both optimal, whatever the oracle's solver does;
  (c) that cut value equals the one of the oracle's cut (Dinic, oracle/lexp_oracle.c);
  (d) the same cut: the device's mask equals the oracle's (SOURCE = the sink cannot be reached = takes the proposal, which is the same set
      for every maximum flow).
Tolerances are relative to the max-flow part `mf`, never to konst, which sums a unary cost over every node.

Designed scenes are exact: constant-disparity labels, an edge-only guide (epsilon = 0, omega = 4: a 0 / 255 edge has a coefficient of exactly 0,
a zero-capacity wall; equal guide values have exactly 1) and a proposal whose disparity is out of range at every pixel (proposal cost exactly
COST_FOR_INVALID), with the current cost set to COST_FOR_INVALID + (wanted net terminal capacity - pairwise part).  Every capacity, push and
sum is then a small dyadic number: flows, konst and cut values must agree exactly and the masks must be identical.
(Sorted after the other graph-cut tests of the -m gpu suite.)"""
import math

import numpy as np
import pytest

from oracle import lexp_oracle as O
from lexp_replay import REPORT, U, certify_gc_step, proposal_costs
from lexp_testlib import TorchDeviceMemory, bits, seeded_labels

pytestmark = pytest.mark.gpu

INVALID = O.COST_FOR_INVALID
FAR = np.array([0, 0, -4, 0], np.float32)     # disparity -4 < MIN_DISPARITY everywhere: proposal cost exactly COST_FOR_INVALID
LAM, TH = 2.0, 1.5                            # designed scenes: c01 = c10 = LAM * TH = 3 between FAR and any label below, c00 in {0, 1, 2}
LEVELS = (3.0, 3.25, 3.5)                     # disparities of the designed scenes' current labels


@pytest.fixture(scope="module")
def devmem():
    return TorchDeviceMemory()


def make_energy(guide, D=8, seed=0, windR=8):
    """Both views on the same guide (uint8 [H][W] or [H][W][3]) and synthetic volumes."""
    import localexpstereo_b200 as L
    img = np.ascontiguousarray(guide if guide.ndim == 3 else np.repeat(guide[..., None], 3, axis=2), np.uint8)
    H, W = img.shape[:2]
    return L.CostVolumeEnergy(img, img, O.synthetic_volume(D, H, W, 1234 + seed), O.synthetic_volume(D, H, W, 1235 + seed),
                              L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5), D - 1)


def make_plan(E, regions):
    from localexpstereo_b200.sweep import window_rects
    plan = E.make_plan(window_rects(regions, E.params.windR, E.width, E.height), regions)
    plan.set_units(regions, np.arange(len(regions)))
    return plan


# ---- designed (exact) scenes ---------------------------------------------------------------------------------------------------------
def level_labels(levels):
    """Constant-disparity labels from a map of disparities."""
    lab = np.zeros(levels.shape + (4,), np.float32)
    lab[..., 2] = levels
    return lab


def designed_state(E, plan, regions, tr_want, labels, mode, devmem, plane=FAR):
    """pm_begin a state under which every cell's graph has the net terminal capacities tr_want (dyadic, float32 [H][W]): the proposal
    costs exactly COST_FOR_INVALID, so with cur = q the first add_tweights leaves tr = 0 and the rest is the pairwise part tr0; add_tweights
    is additive, so cur = q + (tr_want - tr0) gives tr_want.  Returns the proposals."""
    H, W = E.height, E.width
    planes = np.tile(plane, (len(regions), 1))
    E.set_smoothness(LAM, 4.0, TH, 0.0)
    E.pm_begin(mode, np.full((H, W), INVALID, np.float32), labels)
    coeff = E.smooth_coeff(mode)
    assert np.isin(coeff, (0.0, 1.0)).all()
    q = proposal_costs(E, plan, planes, mode, devmem)
    cost = np.full((H, W), INVALID, np.float32)
    for (x, y, w, h) in regions:
        sl = np.s_[y:y + h, x:x + w]
        assert (q[sl] == INVALID).all()
        tr0, _, _ = O.expansion_graph(cost, labels, q[sl], plane, (x, y, w, h), coeff, LAM, TH)
        cost[sl] = INVALID + (tr_want[sl] - tr0)
        assert np.array_equal(cost[sl].astype(np.float64) - float(INVALID), tr_want[sl].astype(np.float64) - tr0)
    E.pm_begin(mode, cost, labels)
    for (x, y, w, h) in regions:
        sl = np.s_[y:y + h, x:x + w]
        assert np.array_equal(O.expansion_graph(cost, labels, q[sl], plane, (x, y, w, h), coeff, LAM, TH)[0], tr_want[sl])
    return planes


def random_design(rng, H, W, block=3, wall=0.4, spread=12):
    """An edge-only guide of random 0 / 255 blocks (zero-capacity walls along their edges), labels of random disparity levels per 2 x 2
    block, and net terminal capacities in 0.25 * [-spread, spread]."""
    g = (rng.random(((H + block - 1) // block, (W + block - 1) // block)) < wall).astype(np.uint8) * 255
    guide = np.kron(g, np.ones((block, block), np.uint8))[:H, :W]
    lv = np.asarray(LEVELS, np.float32)[rng.integers(0, len(LEVELS), ((H + 1) // 2, (W + 1) // 2))]
    labels = level_labels(np.kron(lv, np.ones((2, 2), np.float32))[:H, :W])
    tr = (rng.integers(-spread, spread + 1, (H, W)) * 0.25).astype(np.float32)
    return guide, labels, tr


def run_designed(E, regions, tr_want, labels, mode, devmem):
    plan = make_plan(E, regions)
    try:
        planes = designed_state(E, plan, regions, tr_want, labels, mode, devmem)
        return certify_gc_step(E, plan, regions, mode, LAM, TH, devmem, planes=planes, exact=True)
    finally:
        plan.close()


def final_state(E, mode, cells):
    c, l = E.pm_get(mode)
    return dict(cost=c, label=l, cells=cells)


GEOMETRY_PLANS = (
    # 1 x 1, 2 x 2, k x 1 and 1 x k cells at the corners, along every edge and inside
    [(0, 0, 1, 1), (32, 0, 2, 2), (0, 21, 1, 5), (28, 25, 6, 1), (8, 0, 7, 1), (0, 8, 1, 6), (33, 7, 1, 5), (10, 25, 7, 1), (6, 6, 2, 2),
     (12, 10, 1, 1), (16, 4, 1, 6), (20, 12, 7, 1), (4, 16, 3, 3)],
    [(0, 0, 9, 7), (25, 0, 9, 6), (0, 20, 10, 6), (25, 19, 9, 7)],                  # corner cells: boundary terms clipped on two sides
    [(11, 0, 10, 5), (0, 9, 6, 7), (28, 8, 6, 9), (12, 22, 9, 4), (11, 9, 9, 8)],   # edge cells and one inner cell
    [(0, 0, 34, 26)],                                                               # the whole image: no boundary terms
)


def scene_geometry(devmem, mode=0, seed=5):
    rng = np.random.default_rng(seed + mode)
    guide, labels, _ = random_design(rng, 26, 34)
    E = make_energy(guide, seed=seed)
    try:
        cells = []
        for regions in GEOMETRY_PLANS:
            cells += run_designed(E, regions, random_design(rng, 26, 34)[2], labels, mode, devmem)
        return final_state(E, mode, cells)
    finally:
        E.close()


def corridor(w, h):
    """A serpentine path through a w x h cell, one pixel wide, inside a one-pixel wall margin.  Every arc of the expansion graph points
    forward in raster order (GE, EG, LG, GG), so the path is a Z: right along a row, then down-left along a diagonal to the next row."""
    path, y = [], 1
    while True:
        path += [(x, y) for x in range(1, w - 1)]
        if y + (w - 3) > h - 2:
            return path
        path += [(w - 2 - t, y + t) for t in range(1, w - 3)]
        y += w - 3


def corridor_scene(w, h):
    """(guide, regions, tr, labels, path) of scene_corridor."""
    H, W = h + 2, 2 * w + 3
    regions = [(1, 1, w, h), (w + 2, 1, w, h)]
    path = corridor(w, h)
    guide = np.full((H, W), 255, np.uint8)
    tr = np.full((H, W), -64.0, np.float32)
    for (rx, ry, _, _), (a, b) in zip(regions, ((8.0, -5.0), (5.0, -8.0))):
        for (x, y) in path:
            guide[ry + y, rx + x] = 0
            tr[ry + y, rx + x] = 0.0
        tr[ry + path[0][1], rx + path[0][0]] = a
        tr[ry + path[-1][1], rx + path[-1][0]] = b
    return guide, regions, tr, level_labels(np.full((H, W), 3.0, np.float32)), path


def scene_corridor(devmem, w=40, h=800, mode=0):
    """Two cells, each one corridor between zero-capacity walls (walls: sink capacity 64, no excess), arcs of 6 along it.  Cell A: excess 8
    at the start, sink capacity 5 at the end -- maximum flow 5, unique minimum cut: the whole corridor takes the proposal.  Cell B: 5 and 8
    -- maximum flow 5 again, unique minimum cut: the corridor keeps its labels.  Both flows travel the whole path."""
    guide, regions, tr, labels, path = corridor_scene(w, h)
    E = make_energy(guide, seed=2)
    try:
        cells = run_designed(E, regions, tr, labels, mode, devmem)
        on = np.zeros((h, w), bool)
        on[tuple(np.array(path).T[::-1])] = True
        assert np.array_equal(cells[0]["mask"], on), "the corridor of cell A must take the proposal, its walls must not"
        assert not cells[1]["mask"].any(), "cell B must keep its labels"
        assert cells[0]["mf"] == cells[1]["mf"] == 5.0
        return final_state(E, mode, cells) | dict(path=len(path))
    finally:
        E.close()


def scene_invalid(devmem, mode=0):
    """COST_FOR_INVALID-dominated cells: current cost 1e6 on the left half of every cell, proposals invalid on a band of rows or columns,
    both invalid on a block of 8 nodes per cell (konst > 8e6), max flow O(10)."""
    import localexpstereo_b200 as L
    H, W = 48, 72
    E = make_energy(O.synthetic_image(H, W, 11), D=12, seed=4)
    lam, th = 0.6, 1.0
    try:
        E.set_smoothness(lam, 10.0, th, 0.01)
        regions = [(2, 2, 32, 32), (38, 2, 32, 20), (38, 25, 30, 20)]
        planes = np.array([[0.02, 0.4, -1.5 - 0.4 * 2, 0], [0.4, 0.03, -1.5 - 0.4 * 38, 0], [0.4, -0.02, -1.5 - 0.4 * 38, 0]], np.float32)
        plan = make_plan(E, regions)
        q = proposal_costs(E, plan, planes, mode, devmem)
        rng = np.random.default_rng(9)
        cost = (0.2 + 0.6 * rng.random((H, W))).astype(np.float32)
        for (x, y, w, h) in regions:
            sl = np.s_[y:y + h, x:x + w]
            qs, cs = q[sl], cost[sl]
            bad = qs == INVALID
            assert bad.any() and not bad.all()
            ok = ~bad
            cs[ok] = (qs[ok] * rng.uniform(0.8, 1.25, int(ok.sum()))).astype(np.float32)
            left = np.zeros((h, w), bool)
            left[:, :w // 2] = True
            cs[left & ok] = INVALID
            both = np.argwhere(left & bad)[:8]
            assert len(both) == 8
            cs[tuple(both.T)] = INVALID
        labels = level_labels((2.0 + 6.0 * rng.random((H, W))).astype(np.float32))
        E.pm_begin(mode, cost, labels)
        cells = certify_gc_step(E, plan, regions, mode, lam, th, devmem, planes=planes)
        for c in cells:
            assert c["konst"] >= 8e6 and 0.1 < c["mf"] < 1e3, (c["region"], c["konst"], c["mf"])
            assert c["mask"].any() and not c["mask"].all()
        plan.close()
        return final_state(E, mode, cells)
    finally:
        E.close()


# ---- tests -----------------------------------------------------------------------------------------------------------------------------
def report(what):
    print(f"{what}: {REPORT['moves']} moves so far, worst |(flow - konst) - cut| / max(mf, 1e-3) = {REPORT['worst']:.2e}, "
          f"{REPORT['ties']} nodes cut differently, largest phase-kernel cell {REPORT['phase_nodes']} nodes")


@pytest.mark.parametrize("mode", [0, 1])
def test_lambda_zero_is_the_closed_form(devmem, mode):
    """lambda = 0: no arcs, every node decides alone -- takes the proposal exactly when cur >= q (a tie takes it: BK's free node is
    SOURCE), and the flow is sum min(cur, q).  Cells: cur = +inf (pm_begin's default); proposal invalid on part of the cell (a steep
    plane); cur == q exactly on blocks, and cur == q == 1e6."""
    H, W = 40, 56
    E = make_energy(O.synthetic_image(H, W, 7), D=12, seed=1)
    try:
        E.set_smoothness(0.0, 10.0, 1.0, 0.01)
        regions = [(1, 1, 14, 12), (20, 2, 16, 14), (2, 18, 30, 16)]
        planes = np.array([[0.1, -0.05, 5.0, 0], [-0.08, 0.12, 6.0, 0], [0.6, 0.0, -8.0, 0]], np.float32)
        plan = make_plan(E, regions)
        q = proposal_costs(E, plan, planes, mode, devmem)
        rng = np.random.default_rng(3 + mode)
        cost = np.full((H, W), np.inf, np.float32)
        factor = np.kron(rng.choice(np.float32([0.5, 1.0, 2.0]), (H // 4 + 1, W // 4 + 1)), np.ones((4, 4), np.float32))[:H, :W]
        for (x, y, w, h) in regions[1:]:
            sl = np.s_[y:y + h, x:x + w]
            cost[sl] = q[sl] * factor[sl]
        inv = np.zeros((H, W), bool)
        inv[18:34, 2:32] = q[18:34, 2:32] == INVALID
        assert inv.any() and not inv[18:34, 2:32].all()
        cost[inv & (factor != 1.0)] = (0.3 + 0.5 * rng.random(int((inv & (factor != 1.0)).sum()))).astype(np.float32)
        labels = level_labels((1.0 + 8.0 * rng.random((H, W))).astype(np.float32))
        E.pm_begin(mode, cost, labels)
        cells = certify_gc_step(E, plan, regions, mode, 0.0, 1.0, devmem, planes=planes)
        plan.close()
        for c, (x, y, w, h) in zip(cells, regions):
            cur = cost[y:y + h, x:x + w]
            assert np.array_equal(c["mask"], cur >= c["q"]), c["region"]
            assert c["mf"] == 0.0
            s = math.fsum(np.minimum(cur, c["q"]).astype(np.float64).ravel())
            assert abs(c["flow"] - s) <= 2 * w * h * U * s, (c["region"], c["flow"], s)
        assert np.isinf(cost[1:13, 1:15]).all()
        ties = [int((cost[y:y + h, x:x + w] == c["q"]).sum()) for c, (x, y, w, h) in zip(cells[1:], regions[1:])]
        assert min(ties) > 10 and (cost[inv] == INVALID).any(), ties
    finally:
        E.close()


@pytest.mark.parametrize("mode", [0, 1])
def test_free_nodes_take_the_proposal(devmem, mode):
    """A node the sink cannot reach is SOURCE: a walled block with tr = 0 everywhere (arcs inside, no terminal arc) and a walled single
    pixel with tr = 0 take the proposal; a walled block with only sink capacity keeps its labels; a walled block with one sink node is
    split by the direction of its arcs (the oracle decides).  Around them random terminal capacities."""
    H, W = 30, 40
    rng = np.random.default_rng(17 + mode)
    guide, labels, tr = random_design(rng, H, W, wall=0.0)
    blocks = dict(free=np.s_[5:9, 5:9], sink=np.s_[5:8, 14:19], one=np.s_[14:15, 6:7], split=np.s_[13:17, 14:18])
    for name, sl in blocks.items():
        guide[sl] = 255
        tr[sl] = -1.0 if name == "sink" else 0.0
    tr[15, 15] = -1.0
    E = make_energy(guide, seed=3)
    try:
        region = (2, 2, 34, 24)
        (c,) = run_designed(E, [region], tr, labels, mode, devmem)
        m = np.zeros((H, W), bool)
        m[2:26, 2:36] = c["mask"]
        assert m[blocks["free"]].all() and m[blocks["one"]].all() and not m[blocks["sink"]].any()
        assert m[blocks["split"]].any() and not m[blocks["split"]].all()
    finally:
        E.close()


def test_invalid_dominated_cells(devmem):
    scene_invalid(devmem)
    report("invalid-dominated")


def test_long_residual_path_on_the_one_cta_kernel(devmem, monkeypatch):
    """Two 40 x 800 corridors (32 000 nodes per cell, just under the 32 768-node threshold of the phase kernels): a path of about 1 600
    nodes, so thousands of push / relabel rounds and dozens of global relabellings."""
    monkeypatch.delenv("LEXP_GC_BIG_NODES", raising=False)
    monkeypatch.delenv("LEXP_GC_RELABEL_EVERY", raising=False)
    r = scene_corridor(devmem)
    assert r["path"] > 1500
    report("corridor")


@pytest.mark.parametrize("mode", [0, 1])
def test_cells_at_corners_edges_and_the_whole_image(devmem, mode):
    scene_geometry(devmem, mode)
    report(f"geometry, mode {mode}")


def test_large_cell_on_the_phase_kernels(devmem, monkeypatch):
    """One 200 x 200 cell (40 000 nodes, above the default threshold: no override) with small cells in the same plan: the phase kernels
    with many blocks per cell, the block-wise konst / sink sums and lexp_gc_phase_flows."""
    monkeypatch.delenv("LEXP_GC_BIG_NODES", raising=False)
    H, W = 224, 220
    rng = np.random.default_rng(23)
    guide, labels, tr = random_design(rng, H, W)
    regions = [(0, 0, 200, 200), (202, 0, 8, 10), (202, 12, 1, 1), (0, 202, 30, 20), (40, 202, 1, 9), (205, 205, 15, 19)]
    E = make_energy(guide, seed=6)
    try:
        cells = run_designed(E, regions, tr, labels, 0, devmem)
        REPORT["phase_nodes"] = max(REPORT["phase_nodes"], max(w * h for (_, _, w, h) in regions))
        assert max(w * h for (_, _, w, h) in regions) > 32768
        assert cells[0]["mf"] > 100 and cells[0]["mask"].any() and not cells[0]["mask"].all()
    finally:
        E.close()
    report("phase kernels")


def test_every_move_of_a_natural_scene(devmem):
    """One graph-cut iteration over two layers on the cones crop with the device proposers; every step's planes are the ones the step
    recorded.  FP32 costs can tie: (d) only counts nodes on different sides, (a) to (c) hold on every move."""
    import lexp_golden
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import GCSweep
    G = lexp_golden.load()
    D = G["D"]
    lam, th = 1.0, 1.0
    E = L.CostVolumeEnergy(G["imL"], None, G["volL"], None, L.Parameters(windR=G["windR"], filterName="GF", filter_param1=1e-4, th_col=0.5), D - 1)
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)]]
    S = GCSweep(E, unit_sizes=[6, 18], proposers=props, lam=lam, omega=10.0, th_smooth=th, epsilon=0.01)
    try:
        S.begin()
        S.init(seeded_labels(S, 4))
        n_moves = n_ties = 0
        worst = 0.0
        for g in S.groups:
            for k, kind, m, sd in S.group_steps(g.layer, g.group, 0, 12):
                cells = certify_gc_step(E, g.plan, g.targets, 0, lam, th, devmem, kind=kind, m=m, seed=sd, ties_ok=True)
                n_moves += len(cells)
                n_ties += sum(c["ties"] for c in cells)
                worst = max([worst] + [c["err"] for c in cells])
        print(f"natural scene: {n_moves} moves, worst |(flow - konst) - cut| / max(mf, 1e-3) = {worst:.2e}, "
              f"{n_ties} nodes cut differently from the oracle (ties)")
        assert n_moves > 1000
    finally:
        S.close()
        E.close()
    report("natural scene")


SCENES = dict(invalid=scene_invalid, corridor=lambda devmem: scene_corridor(devmem, 40, 200), geometry=scene_geometry)


def schedule_variants(devmem, monkeypatch, scene, variants):
    """The scene under each (LEXP_GC_RELABEL_EVERY, LEXP_GC_BIG_NODES) setting (read by lexp_create): states bit-identical to the default
    schedule's, masks identical, flows within the tolerance of the certificate."""
    runs = []
    for relabel, big in [(None, None)] + variants:
        for name, v in (("LEXP_GC_RELABEL_EVERY", relabel), ("LEXP_GC_BIG_NODES", big)):
            if v is None:
                monkeypatch.delenv(name, raising=False)
            else:
                monkeypatch.setenv(name, v)
        runs.append(SCENES[scene](devmem))
    ref = runs[0]
    for (relabel, big), r in zip(variants, runs[1:]):
        what = f"{scene}, LEXP_GC_RELABEL_EVERY={relabel}, LEXP_GC_BIG_NODES={big}"
        assert np.array_equal(bits(r["cost"]), bits(ref["cost"])) and np.array_equal(bits(r["label"]), bits(ref["label"])), what
        for a, b in zip(ref["cells"], r["cells"]):
            assert np.array_equal(a["mask"], b["mask"]), (what, a["region"])
            assert abs(a["flow"] - b["flow"]) <= 1e-6 * max(a["mf"], 1e-3) + 2 * a["slack"], (what, a["region"], a["flow"], b["flow"])


@pytest.mark.parametrize("scene", sorted(SCENES))
def test_cut_does_not_depend_on_the_schedule(devmem, monkeypatch, scene):
    """Global relabelling every 1, 5, 24 (the default) and 4096 rounds, and every cell on the phase kernels (LEXP_GC_BIG_NODES = 0, which
    DESIGN.md section 3d states gives the one-CTA kernel's state bit for bit; the flows are summed in another order)."""
    schedule_variants(devmem, monkeypatch, scene, [("1", None), ("5", None), ("4096", None), (None, "0")])
