"""The call schedule of one local-expansion sweep over one view, as the reference issues it
(FastGCStereo::localExpansionMovesForLayer_CPU, FastGCStereo.h:22-72): for each layer, for each
of its <= 16 disjoint groups (sequential), for each proposal step k (sequential), ONE batched
evaluation of all cells of the group (the `omp parallel for` axis, :30-31).

Multi-GPU: the cells of every group are dealt round-robin to ranks (cell-shard path,
SURVEY.md section 8e); each rank owns a plan per (layer, group) for its own cells only."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List

import numpy as np

from .energy import CostVolumeEnergy, LayerManager, Plan


def v3_layer_units(width):  # main.cpp:395-397
    return [int(width * 0.01), int(width * 0.03), int(width * 0.09)]


V3_STEPS = [9, 3, 3]  # Exp(1)+Ransac(1)+Random(7) | Exp(2)+Ransac(1) | same (main.cpp:391-397)


def shard_cells(cells, rank, world):
    """Cell-shard rule (SURVEY.md section 8e): the cells of one disjoint group are dealt round-robin to ranks."""
    return np.asarray(cells, dtype=np.int64)[rank::world]


def tile_offsets(target_rects):
    """Float offsets of the per-cell unary tiles inside a rank's contiguous tile buffer (the all-gather payload,
    same rule as lexp_plan_eval_device_tiles): tile i starts at the sum of the areas of tiles 0..i-1."""
    areas = np.array([r[2] * r[3] for r in target_rects], dtype=np.int64)
    return np.concatenate([[0], np.cumsum(areas)[:-1]]) if len(areas) else np.zeros(0, np.int64), int(areas.sum())


def window_rects(units, windR, width, height):
    """unit +- windR clipped to the image: the filterRegion initCurrentFast gives a unit region (FastGCStereo.h:101-113)."""
    out = []
    for (x, y, w, h) in units:
        x0, y0, x1, y1 = max(x - windR, 0), max(y - windR, 0), min(x + w + windR, width), min(y + h + windR, height)
        out.append((x0, y0, x1 - x0, y1 - y0))
    return out


@dataclass
class GroupPlan:
    layer: int
    group: int
    cells: np.ndarray        # indices (into the layer's cell list) evaluated by THIS rank
    plan: Plan
    n_steps: int
    units: list              # unit, target and filter rects of those cells and their global ids, in call order
    targets: list
    filters: list
    ids: np.ndarray


def group_plan(energy, lm, li, gi, cells, n_steps=0):
    """The plan of `cells` of layer li (global cell ids: the cells of the layers before it first, layer after layer)."""
    lay = lm.layers[li]
    us, ts, fs = ([rects[r] for r in cells] for rects in (lay.unitRegions, lay.sharedRegions, lay.filterRegions))
    ids = sum(len(l.unitRegions) for l in lm.layers[:li]) + cells
    return GroupPlan(li, gi, cells, energy.make_plan(fs, ts), n_steps, us, ts, fs, ids)


class UnarySweep:
    def __init__(self, energy: CostVolumeEnergy, unit_sizes=None, steps=None, rank=0, world=1):
        self.energy = energy
        self.unit_sizes = unit_sizes or v3_layer_units(energy.width)
        self.steps = steps or V3_STEPS
        self.lm = LayerManager(energy.width, energy.height, energy.params.windR)
        self.groups: List[GroupPlan] = []
        self.total_filter_px = 0     # sum over the WHOLE sweep (all ranks): evals
        self.total_target_px = 0
        self.local_filter_px = 0
        self.local_target_px = 0
        self.local_alg_bytes = 0
        for li, u in enumerate(self.unit_sizes):
            lay = self.lm.addLayer(u)
            K = self.steps[li]
            for gi, cells in enumerate(lay.disjointRegionSets):
                cells = np.asarray(cells, dtype=np.int64)
                self.total_filter_px += K * sum(lay.filterRegions[r][2] * lay.filterRegions[r][3] for r in cells)
                self.total_target_px += K * sum(lay.sharedRegions[r][2] * lay.sharedRegions[r][3] for r in cells)
                mine = shard_cells(cells, rank, world)
                if len(mine) == 0:
                    continue
                g = group_plan(energy, self.lm, li, gi, mine, K)
                self.groups.append(g)
                self.local_filter_px += K * g.plan.filter_px
                self.local_target_px += K * g.plan.target_px
                self.local_alg_bytes += K * g.plan.algorithmic_bytes
        self.launches_per_sweep = sum(g.n_steps for g in self.groups)

    def layer(self, li):
        return self.lm.layers[li]

    def close(self):
        for g in self.groups:
            g.plan.close()
        self.groups = []


# ---------------------------------------------------------------------------------------------------------------------
# PatchMatch phase on the device: FastGCStereo::run's pmInit iterations (FastGCStereo.h:143-157), i.e. the same call
# schedule with doGC == false, proposals drawn and currentCost_/currentLabeling_ updated on the device (lexp_plan_pm_step).
# ---------------------------------------------------------------------------------------------------------------------
from .energy import PROP_EXPANSION, PROP_LIST, PROP_RANDOM, PROP_RANSAC  # noqa: E402

# The reference's proposer lists (main.cpp:300-306 and 391-397): {Expansion(1), Ransac(1), Random(7)} / {Expansion(2), Ransac(1)} x 2,
# K = 9 / 3 / 3 evaluations per cell visit.  The RansacProposer runs on the device (PROP_RANSAC, DESIGN.md section 3f).
V3_PROPOSERS_REFERENCE = [[(PROP_EXPANSION, 1), (PROP_RANSAC, 1), (PROP_RANDOM, 7)], [(PROP_EXPANSION, 2), (PROP_RANSAC, 1)], [(PROP_EXPANSION, 2), (PROP_RANSAC, 1)]]
# The default schedule of the sweeps and of bench.py: the same K with the RansacProposer slot given to one more RandomProposer draw.
V3_PROPOSERS_DEVICE = [[(PROP_EXPANSION, 1), (PROP_RANDOM, 8)], [(PROP_EXPANSION, 2), (PROP_RANDOM, 1)], [(PROP_EXPANSION, 2), (PROP_RANDOM, 1)]]


def check_proposers(proposers, world):
    """The lists lexp_pm_sweep_create accepts: Expansion, Random and RANSAC slots with K >= 0.  PROP_RANSAC is supported with K = 1
    on one GPU: RansacProposer::startIterations takes a snapshot that later proposals of the same visit would still fit, and the
    multi-GPU cell shard has no RANSAC support."""
    for layer in proposers:
        for kind, K in layer:
            if kind not in (PROP_EXPANSION, PROP_RANDOM, PROP_RANSAC) or K < 0:
                raise ValueError(f"proposer slot ({kind}, {K}): the sweeps run Expansion, Random and RANSAC slots with K >= 0")
            if kind == PROP_RANSAC and K != 1:
                raise ValueError("PROP_RANSAC with K != 1: later proposals would need the snapshot of startIterations, which is not kept")
            if kind == PROP_RANSAC and world != 1:
                raise ValueError("PROP_RANSAC with world > 1: the multi-GPU cell shard has no RANSAC support")


def pm_seed(base, mode, iteration, layer, group, step):
    """Random stream of one launch = one (view, iteration, layer, group, proposal step); the kernel hashes it with the cell id."""
    M = 0xFFFFFFFFFFFFFFFF
    z = (int(base) * 0x9E3779B97F4A7C15 + (mode + 1) * 0xD1B54A32D192ED03 + (iteration + 1) * 0x8CB92BA72F3D8DD7
         + (layer + 1) * 0xABC98388FB8FAC03 + (group + 1) * 0x2545F4914F6CDD1D + (step + 1) * 0xDA942042E4DD58B5) & M
    z = ((z ^ (z >> 33)) * 0xFF51AFD7ED558CCD) & M
    return z ^ (z >> 29)


RUN_INIT, RUN_PM, RUN_GC = 0, 1, 2   # phases of a run (lexp_run_seed)


def run_seed(base, mode, phase, iteration=0):
    """Seed of one phase of a whole run (= lexp_run_seed): RUN_INIT (the random start's seed; iteration ignored), RUN_PM / RUN_GC (the
    base seed of pm / graph-cut iteration `iteration`, which pm_seed then hashes per launch)."""
    M = 0xFFFFFFFFFFFFFFFF
    z = (int(base) * 0x9E3779B97F4A7C15 + (mode + 1) * 0xC2B2AE3D27D4EB4F + (phase + 1) * 0x165667B19E3779F9
         + (0 if phase == RUN_INIT else iteration + 1) * 0x27D4EB2F165667C5) & M
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
    return z ^ (z >> 31)


def expand_proposers(proposers, outer_iter, max_disp, min_disp=0.0):
    """[(kind, K)] -> the proposal steps [(kind, m)] of one cell visit, as the `while (prop->isContinued())` loops of
    FastGCStereo.h:41-46 produce them; RandomProposer stops early when its disparity perturbation width falls below 0.1
    (Proposer.h:149-152) and uses m = outerIter + iter (:124)."""
    steps = []
    for kind, K in proposers:
        for it in range(K):
            if kind == PROP_RANDOM and np.float32(max_disp - min_disp) * np.float32(0.5) ** (outer_iter + it + 1) < 0.1:
                break
            steps.append((kind, outer_iter + it if kind == PROP_RANDOM else 0))
    return steps


def pm_schedule(lm: LayerManager, unit_sizes, world):
    """The (layer, group) sequence of one pm iteration on a `world`-rank cell shard, identical on every rank:
    [(layer, group, cells_by_rank, owners)] with cells_by_rank[r] = the cells rank r evaluates (round-robin deal of the group's
    cells, SURVEY.md 8e) and owners = the ranks that own at least one cell.  Adds the layers to `lm`."""
    out = []
    for li, u in enumerate(unit_sizes):
        lay = lm.addLayer(u)
        for gi, cells in enumerate(lay.disjointRegionSets):
            by_rank = [shard_cells(cells, r, world) for r in range(world)]
            out.append((li, gi, by_rank, [r for r in range(world) if len(by_rank[r])]))
    return out


class EpochClock:
    """Host-side bookkeeping of the group epochs of the multi-GPU cell shard (lexp_plan_pm_step_ex).  Groups are numbered
    1, 2, ... identically on every rank; `rel` counts the groups issued since the device-side epoch base was last advanced
    (once per init / iteration, so that an iteration's launches carry the same relative numbers every time and can be replayed
    as a CUDA graph); last_rel[r] is the last epoch rank r published, relative to the current base (None: never)."""

    def __init__(self, rank, world):
        self.rank, self.world, self.rel, self.last_rel, self.base = rank, world, 0, [None] * 8, 0

    def sync_args(self, first, last):
        """publish_epoch / wait_epochs / wait_mask of one step of the group being issued (relative epoch rel + 1)."""
        a = {"publish_epoch": self.rel + 1 if last else 0}
        if first:   # including this rank's own previous groups: the launches of an iteration overlap on the device
            a["wait_epochs"] = [0 if e is None else e for e in self.last_rel]
            a["wait_mask"] = sum(1 << r for r, e in enumerate(self.last_rel) if e is not None)
        return a

    def group_done(self, owners):
        self.rel += 1
        for r in owners:
            self.last_rel[r] = self.rel

    def advance(self):
        """All groups of an init / iteration have been issued: returns the delta for lexp_pm_advance_epoch."""
        delta = self.rel
        self.last_rel = [None if e is None else e - delta for e in self.last_rel]
        self.base += delta
        self.rel = 0
        return delta


class PMSweep:
    """Device-resident PatchMatch phase of one view: state (currentCost_, currentLabeling_) in HBM, one plan per (layer, group),
    one launch per proposal step; nothing crosses PCIe between `begin` / `init` and `get`.

    Multi-GPU cell shard (rank / world): the cells of every group are dealt round-robin to ranks; every rank holds a full copy of
    the state and, after `connect` / `connect_local`, its kernels store accepted updates into all copies.  Groups are numbered
    by epochs (the same on every rank, whether it owns cells of a group or not): the last step of a group publishes the epoch,
    the first step of the next group a rank takes part in waits for the latest epoch of every rank that has published one."""

    def __init__(self, energy: CostVolumeEnergy, unit_sizes=None, proposers=None, rank=0, world=1, mode=0):
        self.energy, self.mode, self.rank, self.world = energy, mode, rank, world
        self.unit_sizes = unit_sizes or v3_layer_units(energy.width)
        self.proposers = proposers or V3_PROPOSERS_DEVICE
        check_proposers(self.proposers, world)
        self.lm = LayerManager(energy.width, energy.height, energy.params.windR)
        self.groups: List[GroupPlan] = []          # this rank's plans
        self.schedule = []                         # every (layer, group) in order: (GroupPlan or None, [ranks that own cells])
        for (li, gi, by_rank, owners) in pm_schedule(self.lm, self.unit_sizes, world):
            gp = None
            if len(by_rank[rank]):
                gp = group_plan(energy, self.lm, li, gi, by_rank[rank])
                gp.plan.set_units(gp.units, gp.ids)
                self.groups.append(gp)
            self.schedule.append((li, gi, gp, owners))
        # initCurrentFast (FastGCStereo.h:101-113): every unit region of layer 0 with filterRegion = unit +- windR
        n0 = len(self.lm.layers[0].unitRegions)
        self.init_owners = [r for r in range(world) if len(range(r, n0, world))]
        self.init_index = np.arange(n0)[rank::world]          # which of the layer-0 units this rank initialises
        self.init_units = [self.lm.layers[0].unitRegions[r] for r in self.init_index]
        self.init_group = self.init_plan = None       # the initialisation's GroupPlan and its Plan
        if len(self.init_units):
            fr = window_rects(self.init_units, energy.params.windR, energy.width, energy.height)
            self.init_group = GroupPlan(0, 0, self.init_index, energy.make_plan(fr, self.init_units), 0, self.init_units, self.init_units,
                                        fr, self.init_index)
            self.init_plan = self.init_group.plan
            self.init_plan.set_units(self.init_units, self.init_index)
        self.clock = EpochClock(rank, world)

    # ---- multi-GPU wiring (after begin(): the state must exist) ------------------------------------------------------------
    def connect(self, all_handles):
        self.energy.pm_ipc_connect(self.rank, self.world, all_handles, self.mode)

    def connect_local(self, peer_energies):
        self.energy.pm_connect_local(self.rank, peer_energies, self.mode)

    def _advance(self):
        """All groups of an init / iteration have been issued: move the device epoch base past them."""
        self.energy.pm_advance_epoch(self.clock.advance(), self.mode)

    def begin(self, cost=None, labeling=None):
        self.energy.pm_begin(self.mode, cost, labeling)

    # ---- the schedule ----------------------------------------------------------------------------------------------------------
    def group_steps(self, layer, group, iteration, seed):
        """The proposal steps of one visit of (layer, group) in pm / graph-cut iteration `iteration`: [(index, kind, m, seed)], the
        seed being the launch's random stream."""
        E = self.energy
        return [(k, kind, m, pm_seed(seed, self.mode, iteration, layer, group, k))
                for k, (kind, m) in enumerate(expand_proposers(self.proposers[layer], iteration, E.MAX_DISPARITY, E.MIN_DISPARITY))]

    def walk(self, iteration, seed, issue):
        """The PatchMatch-phase walk of the initialisation (iteration None: one PROP_LIST step of init_group) or of one pm iteration.
        For every group in order it calls issue(group_plan, [(index, kind, m, seed, sync)]) when this rank owns cells of the group,
        sync being the step's publish_epoch / wait_epochs / wait_mask; then it marks the group done and yields the number of steps
        issued.  A group whose proposers all stop early publishes nothing on any rank; a rank without cells of a group still counts
        it.  The launch-chain sync is reset once, before the first group, so all launches of the walk form one chain; the epoch base
        advances once the walk is exhausted."""
        self.energy.pm_reset_sync()
        groups = [(0, 0, self.init_group, self.init_owners)] if iteration is None else self.schedule
        for (li, gi, g, owners) in groups:
            steps = [(0, PROP_LIST, 0, 0)] if iteration is None else self.group_steps(li, gi, iteration, seed)
            if g is not None:
                issue(g, [(k, kind, m, sd, self.clock.sync_args(k == 0, k == len(steps) - 1)) for (k, kind, m, sd) in steps])
            self.clock.group_done(owners if steps else [])
            yield len(steps) if g is not None else 0
        self._advance()

    def init(self, labels):
        """labels [this rank's units of layer 0][4] (all units at world == 1): `currentLabeling(unit) = label;
        ComputeUnaryPotential(unit +- R, unit, ...)` (:107-111)."""
        def issue(g, steps):
            g.plan.pm_step(0, PROP_LIST, planes=labels, init=True, mode=self.mode, **steps[0][4])
        for _ in self.walk(None, 0, issue):
            pass

    def iteration(self, iteration, seed, planes_out=None):
        """One pm iteration over all layers (FastGCStereo.h:153-157).  planes_out: optional {(layer, group): device pointer of
        [steps][n] planes}.  Returns the number of launches."""
        return sum(self.iteration_by_group(iteration, seed, planes_out))

    def iteration_by_group(self, iteration, seed, planes_out=None):
        """Generator form of `iteration`: issues one (layer, group) per step and yields its number of launches (lets a
        single-process test interleave several ranks)."""
        def issue(g, steps):
            for k, kind, m, sd, sync in steps:
                out = 0 if planes_out is None else planes_out[(g.layer, g.group)] + k * g.plan.num_calls * 16
                g.plan.pm_step(k, kind, m, sd, d_planes_out=out, mode=self.mode, **sync)
        return self.walk(iteration, seed, issue)

    def get(self, out_cost=None, out_labeling=None):
        return self.energy.pm_get(self.mode, out_cost=out_cost, out_labeling=out_labeling)

    def close(self):
        for g in self.groups:
            g.plan.close()
        if self.init_plan is not None:
            self.init_plan.close()
        self.groups = []


class GCSweep(PMSweep):
    """The graph-cut iterations of FastGCStereo::run (FastGCStereo.h:171-184: localExpansionMovesForLayer_CPU with doGC == true) on
    the same device-resident state and the same (layer, group, proposal step) schedule as the PatchMatch phase: every step is
    proposals -> ComputeUnaryPotential -> expansionMoveBK (pairwise terms, graph, minimum cut) -> copyTo / setTo, all on the device
    (Plan.gc_step); the steps are ordered by the stream.  Single-GPU (the cell shard of the PatchMatch phase is not wired here).
    `begin` / `init` / `iteration` (pm iterations) are inherited; `gc_iteration` is one iteration of the main loop."""

    def __init__(self, energy: CostVolumeEnergy, unit_sizes=None, proposers=None, mode=0, lam=1.0, omega=10.0, th_smooth=1.0, epsilon=0.01):
        super().__init__(energy, unit_sizes, proposers, 0, 1, mode)
        energy.set_smoothness(lam, omega, th_smooth, epsilon)

    def init(self, labels):
        """initCurrentFast; the image-based energy takes the unary launch + assignment form (lexp_plan_init_step), as the native sweep
        object does for it.  Its pm iterations (`iteration`) run on the PatchMatch-phase kernel like the cost-volume energy's."""
        if getattr(self.energy, "ENERGY_KIND", 0) == 0:
            return super().init(labels)
        if self.init_plan is not None:
            self.init_plan.init_step(labels, mode=self.mode)

    def gc_iteration(self, iteration, seed, planes_out=None, flows_out=None, layers=None):
        """planes_out as PMSweep.iteration; flows_out: optional {(layer, group): device pointer of double [steps][n]} receiving the
        minimum-cut energy of every move; layers: restrict to these layer indices (timing).  Returns the number of proposal steps
        issued."""
        n = 0
        for (li, gi, g, _owners) in self.schedule:
            if layers is not None and li not in layers:
                continue
            for k, kind, m, sd in self.group_steps(li, gi, iteration, seed):
                out = 0 if planes_out is None else planes_out[(li, gi)] + k * g.plan.num_calls * 16
                fl = 0 if flows_out is None else flows_out[(li, gi)] + k * g.plan.num_calls * 8
                g.plan.gc_step(kind, m, sd, d_planes_out=out, d_flows_out=fl, mode=self.mode)
                n += 1
        return n


class NativePMSweep:
    """The same PatchMatch phase driven by the library's own schedule object (lexp_pm_sweep_*: what the C++ adapter
    CudaCostVolumeEnergy::PatchMatchPhase calls): one C call per initialisation / iteration instead of one per proposal step."""

    def __init__(self, energy: CostVolumeEnergy, unit_sizes=None, proposers=None, rank=0, world=1, mode=0):
        import ctypes as C
        from ._capi import check, lib
        self.energy, self.mode = energy, mode
        units = np.ascontiguousarray(unit_sizes or v3_layer_units(energy.width), dtype=np.int32)
        props = proposers or V3_PROPOSERS_DEVICE
        n_prop = np.ascontiguousarray([len(p) for p in props], dtype=np.int32)
        kinds = np.ascontiguousarray([k for p in props for k, _ in p], dtype=np.int32)
        Ks = np.ascontiguousarray([K for p in props for _, K in p], dtype=np.int32)
        h = C.c_void_p()
        check(lib().lexp_pm_sweep_create(energy._h, mode, len(units), units.ctypes.data, n_prop.ctypes.data, kinds.ctypes.data, Ks.ctypes.data,
                                         rank, world, C.byref(h)))
        self._h = h
        self.num_init_labels = lib().lexp_pm_sweep_num_init_labels(self._h)

    def begin(self, cost=None, labeling=None):
        self.energy.pm_begin(self.mode, cost, labeling)

    def init(self, labels):
        from ._capi import check, lib
        lb = np.ascontiguousarray(labels, dtype=np.float32)
        assert lb.shape == (self.num_init_labels, 4)
        check(lib().lexp_pm_sweep_init(self._h, lb.ctypes.data))

    def random_start(self, seed):
        """initCurrentFast with an empty labeling (lexp_pm_sweep_init_random): a random plane through a random pixel of every layer-0
        unit, drawn on the device from the stream pm_rng_state(seed, unit index); begin() first."""
        from ._capi import check, lib
        check(lib().lexp_pm_sweep_init_random(self._h, int(seed) & 0xFFFFFFFFFFFFFFFF))

    def iteration(self, iteration, seed):
        import ctypes as C
        from ._capi import check, lib
        n = C.c_int(0)
        check(lib().lexp_pm_sweep_iteration(self._h, int(iteration), int(seed) & 0xFFFFFFFFFFFFFFFF, C.byref(n)))
        return n.value

    def gc_iteration(self, iteration, seed):
        """One iteration of the graph-cut loop (FastGCStereo.h:171-184) on the device; energy.set_smoothness first."""
        import ctypes as C
        from ._capi import check, lib
        n = C.c_int(0)
        check(lib().lexp_pm_sweep_gc_iteration(self._h, int(iteration), int(seed) & 0xFFFFFFFFFFFFFFFF, C.byref(n)))
        return n.value

    def get(self, out_cost=None, out_labeling=None):
        return self.energy.pm_get(self.mode, out_cost=out_cost, out_labeling=out_labeling)

    def close(self):
        from ._capi import lib
        if self._h:
            lib().lexp_pm_sweep_destroy(self._h)
            self._h = None
