"""Graph-cut moves at the sizes FastGCStereo::run uses, the round limit of a move, and coefficient maps in the subnormal range.

Every certified step goes through lexp_replay.certify_gc_step: checks (a) to (d) of tests/test_gpu_zz_gc_moves.py against the exact minimum
cut of the device's own graph, with their tolerances unchanged.  The steps are issued one at a time in the order of the sweep; the ones not
certified run as plain Plan.gc_step calls.

At size (synthetic scenes, lexp_testlib.seeded_labels, V3_PROPOSERS_DEVICE, smoothness of -mode MiddV3: lambda 0.5 (main.cpp:437,493),
omega 10, th 1, eps 0.01).  Which execution form ran a certified step is observed from its launches, not inferred from the cell sizes.
  * 2048 x 1536 x 256, windR 20 (bench.py's scene): initialisation, one pm iteration, then graph-cut iteration 0 with layer-1 groups
    {0, 8, 15} (48 to 63 cells per plan, up to 35 502 nodes) and layer-2 groups {0} and the one of the 354 816-node cell certified, all on
    the phase kernels; the final state equals a twin context's uninterrupted gc_iteration bit for bit.  Then that layer-2 group with
    V3_PROPOSERS_REFERENCE (device RansacProposer moves).
  * 1436 x 992 x 290, windR 20 (Adirondack's shape), after the initialisation: layer-1 groups {0, 15} (one CTA per cell, up to 19 272
    nodes, about 50 cells per launch) and layer-2 groups {0, 15} (phase kernels, up to 149 769 nodes).
  * 3840 x 2160 x 512, windR 32, one view, after the initialisation: the layer-2 group of the 1 215 000-node cell, and the wall time of
    its device steps (2.0 s for the slowest).  Only that group: the scene alone takes 4 minutes, and the file is past 10 with it.
  * The image-based energy of -mode MiddV2 at the demo's geometry (450 x 375, D 64, windR 20, layers 5 / 15 / 25, lambda 20):
    initialisation, two pm iterations, then groups {0, 5, last} of every layer of a graph-cut iteration certified.
FP32 costs of the cost-volume scenes tie at these sizes: there (d) counts the nodes on different sides and (a) to (c) hold on every move.
Each scene prints its moves, largest cell, worst |(flow - konst) - cut| / max(mf, 1e-3), tie nodes, the form and slowest device step of
every layer, and wall time.

Designed scenes (exact; also run on the emulator, tests/test_emu_gc_limits.py):
  * Round limit: the corridor of test_gpu_zz_gc_moves (about 1 600 rounds) under LEXP_GC_MAX_ROUNDS = 0, 24 and 240, one CTA per cell and
    on the phase kernels.  The step returns, lexp_pm_get reports the limit, every pixel holds its old state or the proposal, and both forms
    give the same state and flows bit for bit: they test the limit at the same global relabelling.  lexp_pm_begin clears the report.
  * Many cells on the phase kernels: one plan of 49 designed cells, exact, phase kernels and one CTA per cell bit-identical.
  * Subnormal coefficients: epsilon = 0, omega = 4 and a guide whose neighbour channel-sum differences span about 320 to 430, so that
    exp(-s / omega) runs from normal numbers through the subnormal range to 0.  A flush to zero would turn those capacities into walls.

Measured on an H100 80GB HBM3 (700 W power limit): 2048 x 1536 5 min, 4K 4 min, the rest 3 min 5 s; DESIGN.md section 5 has the numbers."""
import time

import numpy as np
import pytest

from oracle import lexp_oracle as O
from lexp_replay import REPORT, certify_gc_step, proposal_costs
from lexp_testlib import TorchDeviceMemory, bits, energy_and_oracle, make_scene, seeded_labels
import test_gpu_zz_gc_moves as MV

pytestmark = pytest.mark.gpu

MIDDV3 = dict(lam=0.5, omega=10.0, th_smooth=1.0, epsilon=0.01)
BIG_NODES = 32768                  # default LEXP_GC_BIG_NODES: plans with a larger cell run on the phase kernels
FLT_MIN = np.float32(2.0 ** -126)
TINY = 2.0 ** -149                 # the smallest subnormal float


@pytest.fixture(scope="module")
def devmem():
    return TorchDeviceMemory()


class Tally:
    """What a scene prints: moves, largest cell, worst relative duality gap, tie nodes, the slowest device step of every layer and wall
    time; and which execution form ran each layer's certified steps (observed from the launches, lexp_replay.certify_gc_step)."""

    def __init__(self, what):
        self.what, self.moves, self.largest, self.worst, self.ties, self.t0 = what, 0, 0, 0.0, 0, time.perf_counter()
        self.largest_by_layer, self.forms, self.step_s = {}, {}, {}

    def add(self, layer, cells, state):
        self.moves += len(cells)
        n = max(c["region"][2] * c["region"][3] for c in cells)
        self.largest = max(self.largest, n)
        self.largest_by_layer[layer] = max(self.largest_by_layer.get(layer, 0), n)
        self.worst = max([self.worst] + [c["err"] for c in cells])
        self.ties += sum(c["ties"] for c in cells)
        self.forms.setdefault(layer, set()).add("phase" if state["phase"] else "one CTA")
        self.step_s[layer] = max(self.step_s.get(layer, 0.0), state["step_s"])
        if state["phase"]:
            REPORT["phase_nodes"] = max(REPORT["phase_nodes"], n)

    def line(self):
        forms = ", ".join(f"layer {li}: {'/'.join(sorted(f))}, slowest step {self.step_s[li]:.2f} s" for li, f in sorted(self.forms.items()))
        return (f"{self.what}: {self.moves} moves, largest cell {self.largest} nodes, worst |(flow - konst) - cut| / max(mf, 1e-3) = "
                f"{self.worst:.2e}, {self.ties} tie nodes ({forms}), {time.perf_counter() - self.t0:.1f} s")


def largest_cell(g):
    return max(t[2] * t[3] for t in g.targets)


def certify_groups(S, devmem, it, seed, pick, T, ties_ok=False, run_others=True):
    """Graph-cut iteration `it` of the sweep S issued step by step: the steps of the groups with pick(layer, group) are certified, the
    others run uncertified (run_others) or not at all."""
    E = S.energy
    coeff = E.smooth_coeff(S.mode)
    lam, th = S.smooth["lam"], S.smooth["th_smooth"]
    state = {}
    for (li, gi, g, _) in S.schedule:
        chosen = pick(li, gi)
        if not chosen and not run_others:
            continue
        for k, kind, m, sd in S.group_steps(li, gi, it, seed):
            if chosen:
                cells = certify_gc_step(E, g.plan, g.targets, S.mode, lam, th, devmem, kind=kind, m=m, seed=sd, ties_ok=ties_ok, coeff=coeff,
                                        state=state)
                T.add(li, cells, state)
            else:
                g.plan.gc_step(kind, m, sd, mode=S.mode)
                state.clear()
        if chosen:
            print(f"  layer {li} group {gi}: {T.moves} moves so far, {time.perf_counter() - T.t0:.1f} s", flush=True)


def make_sweep(E, proposers, units=None, smooth=MIDDV3):
    from localexpstereo_b200.sweep import GCSweep
    S = GCSweep(E, unit_sizes=units, proposers=proposers, **smooth)
    S.smooth = smooth
    return S


def device_volume(D, H, W, seed=1234):
    import torch
    vol = torch.rand((D, H, W), generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda", dtype=torch.float32)
    torch.cuda.synchronize()   # torch fills the volume on its own stream; the library's stream is non-blocking
    return vol


def volume_energy(img, vol, D, windR):
    import localexpstereo_b200 as L
    return L.CostVolumeEnergy(img, None, vol, None, L.Parameters(windR=windR, filterName="GF", filter_param1=1e-4, th_col=0.5), D - 1)


def layer2_largest(S):
    return max((g for g in S.groups if g.layer == 2), key=largest_cell)


# ---- at size ---------------------------------------------------------------------------------------------------------------------------
def test_benchmark_scene(devmem, monkeypatch):
    """bench.py's scene (2048 x 1536 x 256, windR 20, V3_PROPOSERS_DEVICE, the volume drawn on the device with seed 1234): the
    initialisation and one pm iteration, then graph-cut iteration 0 issued step by step, layer-1 groups {0, 8, 15} (48 to 63 cells of up to
    35 502 nodes per plan) and layer-2 groups {0} and the one of the 354 816-node cell certified, every other group run uncertified.  The
    phase kernels must have run every certified step of layers 1 and 2.  The state at the end must equal a twin context's uninterrupted
    gc_iteration(0) bit for bit.  Then the layer-2 group of the largest cell once more with V3_PROPOSERS_REFERENCE: RansacProposer moves."""
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import V3_PROPOSERS_DEVICE, V3_PROPOSERS_REFERENCE
    monkeypatch.delenv("LEXP_GC_BIG_NODES", raising=False)
    monkeypatch.delenv("LEXP_GC_MAX_ROUNDS", raising=False)
    W, H, D, windR, seed = 2048, 1536, 256, 20, 4321
    img = synth.synthetic_image(H, W, 42)
    vol = device_volume(D, H, W)
    E, Et = volume_energy(img, vol, D, windR), volume_energy(img, vol, D, windR)
    S, St = make_sweep(E, V3_PROPOSERS_DEVICE), make_sweep(Et, V3_PROPOSERS_DEVICE)
    T = Tally(f"{W} x {H} x {D}, windR {windR}")
    try:
        labels = seeded_labels(S, seed)
        for X in (S, St):
            X.begin()
            X.init(labels)
            X.iteration(0, seed)
        t0 = time.perf_counter()
        St.gc_iteration(0, seed + 1)
        Et.sync()
        print(f"  twin: uninterrupted graph-cut iteration {time.perf_counter() - t0:.1f} s", flush=True)
        want = St.get()
        g2 = layer2_largest(S)
        picks = {0: (), 1: (0, 8, 15), 2: (0, g2.group)}
        certify_groups(S, devmem, 0, seed + 1, lambda li, gi: gi in picks[li], T, ties_ok=True)
        got = S.get()
        assert np.array_equal(bits(got[0]), bits(want[0])) and np.array_equal(bits(got[1]), bits(want[1])), \
            "the state after the certified steps differs from the twin's uninterrupted graph-cut iteration"
        print(T.line())
        assert T.forms[1] == T.forms[2] == {"phase"}, T.forms
        assert min(len(g.targets) for g in S.groups if g.layer == 1 and g.group in picks[1]) > 32
        assert T.largest_by_layer[1] > BIG_NODES and T.largest_by_layer[2] == largest_cell(g2) == 354816, T.largest_by_layer
        R = make_sweep(E, V3_PROPOSERS_REFERENCE)
        try:
            Tr = Tally(f"{W} x {H} x {D}, windR {windR}, V3_PROPOSERS_REFERENCE")
            certify_groups(R, devmem, 1, seed + 2, lambda li, gi: li == 2 and gi == g2.group, Tr, ties_ok=True, run_others=False)
            assert Tr.moves > 0 and Tr.forms[2] == {"phase"}
            print(Tr.line())
        finally:
            R.close()
    finally:
        S.close(); St.close()
        E.close(); Et.close()


def scene_groups(devmem, W, H, D, windR, picks, seed):
    """The initialisation, then only the steps of the groups picks = {layer: groups} of graph-cut iteration 0 (a group "largest": the
    layer-2 group that holds the largest cell)."""
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import V3_PROPOSERS_DEVICE
    vol = device_volume(D, H, W)
    E = volume_energy(synth.synthetic_image(H, W, 42), vol, D, windR)
    S = make_sweep(E, V3_PROPOSERS_DEVICE)
    T = Tally(f"{W} x {H} x {D}, windR {windR}")
    try:
        picks = {li: {layer2_largest(S).group if g == "largest" else g for g in gs} for li, gs in picks.items()}
        S.begin()
        S.init(seeded_labels(S, seed))
        certify_groups(S, devmem, 0, seed + 1, lambda li, gi: gi in picks.get(li, ()), T, ties_ok=True, run_others=False)
        print(T.line())
        return T
    finally:
        S.close()
        E.close()
        del vol


def test_adirondack_shape(devmem, monkeypatch):
    monkeypatch.delenv("LEXP_GC_BIG_NODES", raising=False)
    T = scene_groups(devmem, 1436, 992, 290, 20, {1: (0, 15), 2: (0, 15)}, 7)
    assert BIG_NODES > T.largest_by_layer[1] > 15000 and T.largest_by_layer[2] > BIG_NODES, T.largest_by_layer
    assert T.forms == {1: {"one CTA"}, 2: {"phase"}}, T.forms


def test_4k_largest_cell(devmem, monkeypatch):
    """3840 x 2160 x 512, windR 32, one view, after the initialisation: the layer-2 group of the 1 215 000-node cell (its three steps)."""
    monkeypatch.delenv("LEXP_GC_BIG_NODES", raising=False)
    T = scene_groups(devmem, 3840, 2160, 512, 32, {2: ("largest",)}, 8)
    assert T.largest_by_layer[2] == 1215000 and T.forms == {2: {"phase"}}, (T.largest_by_layer, T.forms)


def scene_image_based(devmem, W=450, H=375, D=64, units=(5, 15, 25), pm_iterations=2, seed=8):
    """-mode MiddV2's energy at the demo's geometry: init, pm iterations on the device, then groups {0, 5, last} of every layer of a
    graph-cut iteration certified on the device's own graph (its FP32 unary costs), the other groups run in between."""
    import localexpstereo_b200 as L
    imL, imR, _, _ = make_scene(H, W, D, seed=seed)
    lam = 20.0
    E, _ = energy_and_oracle((imL, imR, None, None), D, 20, naive=True, lambda_=lam)
    props = [[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 1)], [(L.PROP_EXPANSION, 1)]]
    S = make_sweep(E, props, list(units), dict(lam=lam, omega=10.0, th_smooth=1.0, epsilon=0.01))
    T = Tally(f"image-based energy {W} x {H} x {D}, layers {units}")
    try:
        S.begin()
        S.init(seeded_labels(S, seed))
        for it in range(pm_iterations):
            S.iteration(it, seed)
        last = {li: len(lay.disjointRegionSets) - 1 for li, lay in enumerate(S.lm.layers)}
        certify_groups(S, devmem, 0, seed + 1, lambda li, gi: gi in (0, 5, last[li]), T)
        print(T.line())
        return T
    finally:
        S.close()
        E.close()


def test_image_based_energy_at_the_demo_geometry(devmem, monkeypatch):
    monkeypatch.delenv("LEXP_GC_BIG_NODES", raising=False)
    T = scene_image_based(devmem)
    assert T.moves > 1000 and T.largest_by_layer[2] == 75 * 75, (T.moves, T.largest_by_layer)


# ---- the round limit ------------------------------------------------------------------------------------------------------------------
def corridor_at_limit(devmem, w, h, mode=0):
    """The corridor scene under the round limit the environment sets (LEXP_GC_MAX_ROUNDS, read by lexp_create): the step returns,
    lexp_pm_get reports the limit and still copies the state, every pixel of a cell holds its old state or the proposal and nothing
    outside the cells changes.  Then lexp_pm_begin clears the report: a move that needs no push round certifies and lexp_pm_get is
    clean.  Returns the limited step's (cost, label, flows)."""
    import localexpstereo_b200 as L
    guide, regions, tr, labels, path = MV.corridor_scene(w, h)
    E = MV.make_energy(guide, seed=2)
    try:
        plan = MV.make_plan(E, regions)
        planes = MV.designed_state(E, plan, regions, tr, labels, mode, devmem)
        pre_c, pre_l = E.pm_get(mode)
        d_fl = devmem.zeros((len(regions), 2))
        plan.gc_step(L.PROP_LIST, planes=planes, d_flows_out=devmem.ptr(d_fl), mode=mode)
        E.sync()
        post_c, post_l = np.empty_like(pre_c), np.empty_like(pre_l)
        with pytest.raises(L.LexpError, match="round limit"):
            E.pm_get(mode, out_cost=post_c, out_labeling=post_l)
        flows = np.ascontiguousarray(devmem.download(d_fl)).view(np.float64)[:, 0].copy()
        inside = np.zeros(pre_c.shape, bool)
        for (x, y, cw, ch), plane in zip(regions, planes):
            sl = np.s_[y:y + ch, x:x + cw]
            inside[sl] = True
            old = (bits(post_c[sl]) == bits(pre_c[sl])) & (bits(post_l[sl]) == bits(pre_l[sl])).all(axis=2)
            new = (post_c[sl] == O.COST_FOR_INVALID) & (bits(post_l[sl]) == bits(plane)).all(axis=2)
            assert (old | new).all(), f"(a) cell {(x, y, cw, ch)}: a pixel holds neither its old state nor the proposal"
        assert np.array_equal(bits(post_c[~inside]), bits(pre_c[~inside])) and np.array_equal(bits(post_l[~inside]), bits(pre_l[~inside]))
        # lexp_pm_begin (inside designed_state) clears the report; no node holds excess, so the move ends at the first global relabelling
        MV.designed_state(E, plan, regions, np.minimum(tr, 0.0), labels, mode, devmem)
        cells = certify_gc_step(E, plan, regions, mode, MV.LAM, MV.TH, devmem, planes=planes, exact=True)
        assert all(c["mf"] == 0.0 for c in cells)
        E.pm_get(mode)
        plan.close()
        return post_c, post_l, flows
    finally:
        E.close()


def round_limit_forms(devmem, monkeypatch, limits, w, h):
    for limit in limits:
        monkeypatch.setenv("LEXP_GC_MAX_ROUNDS", str(limit))
        runs = []
        for big in (None, "0"):   # one CTA per cell, then every cell on the phase kernels
            if big is None:
                monkeypatch.delenv("LEXP_GC_BIG_NODES", raising=False)
            else:
                monkeypatch.setenv("LEXP_GC_BIG_NODES", big)
            runs.append(corridor_at_limit(devmem, w, h))
        (ca, la, fa), (cb, lb, fb) = runs
        assert np.array_equal(bits(ca), bits(cb)) and np.array_equal(bits(la), bits(lb)), f"limit {limit}: the two forms differ"
        assert np.array_equal(fa.view(np.uint64), fb.view(np.uint64)), (limit, fa, fb)
        print(f"round limit {limit}: flows {fa.tolist()}, {int((ca == O.COST_FOR_INVALID).sum())} pixels at COST_FOR_INVALID")


def test_round_limit(devmem, monkeypatch):
    """Limits 0, 24 and 240; then the whole corridor (about 1 600 rounds) on a context with the default limit certifies exactly."""
    round_limit_forms(devmem, monkeypatch, (0, 24, 240), 40, 800)
    monkeypatch.delenv("LEXP_GC_MAX_ROUNDS")
    monkeypatch.delenv("LEXP_GC_BIG_NODES", raising=False)
    assert MV.scene_corridor(devmem, 40, 800)["path"] > 1500


def scene_many_cells(devmem, n_side=7, cell=6, gap=2):
    """One plan of n_side^2 cells (49 by default: more than 32) of the designed, exact kind, on the phase kernels (LEXP_GC_BIG_NODES = 0)
    and one CTA per cell: both certified with no tolerance and bit-identical.  The first 32 cells hold no excess (they are done at the
    first global relabelling), the others random designs with flow to push: their cuts depend on the phase kernels' per-cell bookkeeping
    (done / active flags, per-block sums) beyond the 32nd cell."""
    import os
    H = W = n_side * (cell + gap) + gap
    rng = np.random.default_rng(41)
    guide, labels, tr = MV.random_design(rng, H, W)
    regions = [(gap + i * (cell + gap), gap + j * (cell + gap), cell, cell) for j in range(n_side) for i in range(n_side)]
    for (x, y, w, h) in regions[:32]:
        tr[y:y + h, x:x + w] = np.minimum(tr[y:y + h, x:x + w], 0.0)
    runs = []
    prev = os.environ.get("LEXP_GC_BIG_NODES")
    try:
        for big in ("0", None):
            if big is None:
                os.environ.pop("LEXP_GC_BIG_NODES", None)
            else:
                os.environ["LEXP_GC_BIG_NODES"] = big
            E = MV.make_energy(guide, seed=12)
            try:
                plan = MV.make_plan(E, regions)
                planes = MV.designed_state(E, plan, regions, tr, labels, 0, devmem)
                state = {}
                cells = certify_gc_step(E, plan, regions, 0, MV.LAM, MV.TH, devmem, planes=planes, exact=True, state=state)
                assert state["phase"] == (big == "0"), state
                plan.close()
                runs.append((state["cost"], state["label"], cells))
            finally:
                E.close()
    finally:
        if prev is None:
            os.environ.pop("LEXP_GC_BIG_NODES", None)
        else:
            os.environ["LEXP_GC_BIG_NODES"] = prev
    (ca, la, xa), (cb, lb, xb) = runs
    assert np.array_equal(bits(ca), bits(cb)) and np.array_equal(bits(la), bits(lb))
    assert all(c["mf"] > 0 for c in xa[32:]) and all(a["flow"] == b["flow"] for a, b in zip(xa, xb))
    return xa


def test_many_cells_on_the_phase_kernels(devmem):
    assert len(scene_many_cells(devmem)) > 32


# ---- subnormal coefficients ------------------------------------------------------------------------------------------------------------
def subnormal_guide(H, W, seed=0):
    """Four colours in a 2 x 2 pattern, all six pairwise channel-sum distances 350 to 400, each channel jittered by up to +-10: every
    forward neighbour pair (GE, EG, LG, GG) joins two different colours, at a distance of about 320 to 430."""
    base = np.array([[0, 0, 0], [200, 175, 0], [200, 0, 175], [0, 175, 200]], np.int32)
    ys, xs = np.mgrid[0:H, 0:W]
    rng = np.random.default_rng(seed)
    img = base[(xs % 2) + 2 * (ys % 2)] + rng.integers(-10, 11, (H, W, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


def check_subnormal_coefficients(E, guide, mode=0):
    """The device's maps against the FP64 exp rounded to float: the same zero pattern, 2e-6 relative above FLT_MIN and 2 ulp of the
    smallest subnormal below it.  Returns the maps."""
    got, want = E.smooth_coeff(mode), O.smoothness_coeff(guide, 4.0, 0.0)
    assert np.array_equal(got == 0, want == 0), f"{int(((got == 0) != (want == 0)).sum())} coefficients differ in being 0"
    sub = (want > 0) & (want < FLT_MIN)
    assert np.abs(got[sub].astype(np.float64) - want[sub]).max() <= 2 * TINY
    norm = want >= FLT_MIN
    assert np.allclose(got[norm], want[norm], rtol=2e-6, atol=0)
    n_norm, n_sub = int((norm & (want < 1e-30)).sum()), int(sub.sum())
    n_zero = int(((want == 0) & (O.smoothness_coeff(np.zeros_like(guide), 4.0, 0.0) != 0)).sum())   # zero inside the image
    assert n_norm > 50 and n_sub > 500 and n_zero > 50, (n_norm, n_sub, n_zero)
    return got


def scene_subnormal(devmem, mode=0, H=40, W=56):
    """epsilon = 0, omega = 4 on subnormal_guide: coefficient maps, pairwise terms bit for bit on the device's own maps, and every move
    of one step certified.  The moves: current cost = proposal cost = COST_FOR_INVALID (FAR plane), constant-disparity labels, so every
    terminal and arc capacity of the graph is a sum of pairwise terms of subnormal size (exact in float).  The oracle's cut has nodes on
    both sides; with the tiny capacities flushed to zero every node would be free and take the proposal.  Here konst is about
    N * COST_FOR_INVALID and every cut value is below 1e-30, so the tolerances of (b) and (c) (1e-9 absolute) say nothing: the operative
    check is (d), the device's mask equal to the oracle's node for node, with the mask assertions below."""
    import localexpstereo_b200 as L
    guide = subnormal_guide(H, W, 3 + mode)
    E = MV.make_energy(guide, seed=9)
    try:
        E.set_smoothness(MV.LAM, 4.0, MV.TH, 0.0)
        E.pm_begin(mode, np.zeros((H, W), np.float32), np.zeros((H, W, 4), np.float32))
        coeff = check_subnormal_coefficients(E, guide, mode)
        rng = O.CvRNG(5)
        lab = np.zeros((H, W, 4), np.float32)
        for y in range(0, H, 4):
            for x in range(0, W, 4):
                lab[y:y + 4, x:x + 4] = O.create_random_label(rng, x, y, 0.0, 7.0)
        E.pm_begin(mode, np.zeros((H, W), np.float32), lab)
        regions = [(6, 5, 20, 18), (0, 0, 5, 4), (W - 9, H - 11, 9, 11), (30, 0, 1, 1)]
        planes = [O.create_random_label(rng, r[0], r[1], 0.0, 7.0) for r in regions]
        for r, pl, g in zip(regions, planes, E.computeSmoothnessTermsExpansion(regions, planes, mode)):
            want = O.smoothness_terms_expansion(lab, pl, r, coeff, MV.LAM, MV.TH)
            for t in range(3):
                for fi, k in enumerate(O.FORWARD):
                    assert np.array_equal(bits(g[t][fi]), bits(want[t][k])), (mode, r, t, k)
        regions = [(1, 1, 24, 20), (28, 2, 26, 16), (3, 24, 40, 14), (46, 22, 9, 17)]
        plan = MV.make_plan(E, regions)
        lv = np.asarray(MV.LEVELS, np.float32)[np.random.default_rng(11 + mode).integers(0, 3, ((H + 1) // 2, (W + 1) // 2))]
        labels = MV.level_labels(np.kron(lv, np.ones((2, 2), np.float32))[:H, :W])
        cost = np.full((H, W), O.COST_FOR_INVALID, np.float32)
        E.pm_begin(mode, cost, labels)
        q = proposal_costs(E, plan, np.tile(MV.FAR, (len(regions), 1)), mode, devmem)
        for (x, y, w, h) in regions:
            assert (q[y:y + h, x:x + w] == O.COST_FOR_INVALID).all()
        cells = certify_gc_step(E, plan, regions, mode, MV.LAM, MV.TH, devmem, planes=np.tile(MV.FAR, (len(regions), 1)), coeff=coeff)
        for c in cells:
            x, y, w, h = c["region"]
            tr, _, cap = O.expansion_graph(cost, labels, c["q"], MV.FAR, c["region"], coeff, MV.LAM, MV.TH)
            small = np.concatenate([np.abs(tr).ravel(), cap.ravel()])
            nz = small[small > 0]
            assert (small < 1e-30).all() and (nz < FLT_MIN).mean() > 0.25, (c["region"], (nz < FLT_MIN).mean())
            assert 0.0 < c["mf"] < 1e-30 and not c["mask"].all() and c["mask"].any(), (c["region"], c["mf"])
        plan.close()
        return E.pm_get(mode)
    finally:
        E.close()


@pytest.mark.parametrize("mode", [0, 1])
def test_subnormal_coefficients_and_moves(devmem, monkeypatch, mode):
    """One CTA per cell, then every cell on the phase kernels: the same state bit for bit."""
    monkeypatch.delenv("LEXP_GC_BIG_NODES", raising=False)
    a = scene_subnormal(devmem, mode)
    monkeypatch.setenv("LEXP_GC_BIG_NODES", "0")
    b = scene_subnormal(devmem, mode)
    assert np.array_equal(bits(a[0]), bits(b[0])) and np.array_equal(bits(a[1]), bits(b[1]))
