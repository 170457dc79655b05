"""Times one pm iteration of the image-based energy (NaiveStereoEnergy, `-mode MiddV2`) on the device and prints one JSON line per
measurement, with the card's name and power limit:
  * the pm iteration (PMSweep.iteration: MiddV2's layers 5 / 15 / 25, the reference's proposer lists V3_PROPOSERS_REFERENCE with the
    RansacProposer slot) -- eager and replayed from a CUDA graph; evals/s counts the filterRect pixels the iteration evaluates;
  * in the same run, the plain unary sweep bench.py reports for this workload (the same 240 batched evaluations with host-supplied
    planes into an H x W image, no proposals and no update) at the same geometry;
  * the reference's pm iteration on the host (oracle/_ref's ref_pm_group per group, its OpenMP loop) where oracle/_ref is built.  It
    has no RansacProposer: that slot is replayed as a list (an evaluation of the same size).  At 2048 x 1536 only the first group of
    every layer runs and the iteration time is extrapolated from them.
Sizes: 450 x 375 x 64 (configs[0]'s shape, synthetic images) and 2048 x 1536 x 256, windR 20.
CUDA events around each device call (median of the repetitions after warm-up).  Usage: python scripts/naive_pm_bench.py [--quick]"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from label_cost_bench import card  # noqa: E402

UNITS = [5, 15, 25]   # main.cpp:304-306
SEED = 4321


def timed(fn, stream, warmup, reps):
    import torch
    s = torch.cuda.ExternalStream(stream)
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        fn()
        b.record(s)
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def pm_evals(S, iteration):
    """filterRect pixels one pm iteration evaluates: every cell of every group, once per proposal step."""
    n = 0
    for (li, gi, g, _) in S.schedule:
        k = len(S.group_steps(li, gi, iteration, SEED))
        n += k * sum(f[2] * f[3] for f in g.filters)
    return n


def device_pm(E, D, quick):
    import torch
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import PMSweep, V3_PROPOSERS_REFERENCE
    S = PMSweep(E, unit_sizes=UNITS, proposers=V3_PROPOSERS_REFERENCE)
    side = torch.cuda.Stream()
    E.set_stream(side.cuda_stream)   # the caller's stream from the start, as bench.py: the capture below only switches to its own
    S.begin()
    S.init(synth.synthetic_planes(list(S.lm.layers[0].unitRegions), 1, D, 99)[0])
    warm = 1 if quick else 3
    for it in range(warm):   # also allocates the RANSAC scratch before the capture
        S.iteration(it, SEED)
    IT = warm
    ms_eager = timed(lambda: S.iteration(IT, SEED), side.cuda_stream, 1, 2 if quick else 5)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g):
            E.set_stream(torch.cuda.current_stream().cuda_stream)
            S.iteration(IT, SEED)
        E.set_stream(side.cuda_stream)

    def replay():
        with torch.cuda.stream(side):
            g.replay()
    ms_graph = timed(replay, side.cuda_stream, 1, 2 if quick else 5)
    S.get()   # raises on an error flag
    evals = pm_evals(S, IT)
    launches = sum(len(S.group_steps(li, gi, IT, SEED)) for (li, gi, gp, _) in S.schedule if gp is not None)
    del g
    S.close()
    return ms_eager, ms_graph, evals, launches


def device_unary(E, D, quick):
    import torch
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import UnarySweep
    U = UnarySweep(E, unit_sizes=UNITS)
    per_layer = [synth.synthetic_planes(U.layer(li).unitRegions, U.steps[li], D, 7 + li) for li in range(len(U.steps))]
    planes = [torch.from_numpy(np.ascontiguousarray(per_layer[g.layer][:, g.cells, :])).cuda() for g in U.groups]
    out = torch.zeros((E.height, E.width), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    E.set_overlap(True)

    def sweep():
        for gi, g in enumerate(U.groups):
            for k in range(g.n_steps):
                g.plan.eval_device(planes[gi].data_ptr() + k * g.plan.num_calls * 16, out.data_ptr(), E.width * 4, True, 0,
                                   planes_on_device=True)
    ms = timed(sweep, E.stream, 1 if quick else 3, 2 if quick else 5)
    E.set_overlap(False)
    evals = U.total_filter_px
    U.close()
    return ms, evals


def reference_pm(imL, imR, W, H, D, windR, sample_groups):
    """The reference's pm iteration on the host: ref_pm_group per group (RANSAC slot replayed as a list).  sample_groups: run only
    group 0 of each layer and scale by the layer's number of groups."""
    from oracle import lexp_oracle as O
    from oracle import ref_binding as R
    from localexpstereo_b200 import synth
    from localexpstereo_b200.sweep import V3_PROPOSERS_REFERENCE
    ref = R.RefEnergy(imL, imR, windR=windR, eps=1e-4, th_col=10.0, th_grad=2.0, alpha=0.9, max_disp=D - 1.0, kind=1)
    cost, lab = np.full((H, W), np.inf, np.float32), np.zeros((H, W, 4), np.float32)
    lay0 = O.make_layer(W, H, windR, UNITS[0])
    ref.pm_init(lay0["unit"], synth.synthetic_planes([tuple(u) for u in lay0["unit"]], 1, D, 99)[0], windR, cost, lab)
    total, ran = 0.0, 0
    for li, u in enumerate(UNITS):
        lay = O.make_layer(W, H, windR, u)
        props = [(0 if k == 3 else k, K) for k, K in V3_PROPOSERS_REFERENCE[li]]   # PROP_RANSAC -> replayed list
        n_list = sum(K for k, K in props if k == 0)
        groups = [g for g in lay["groups"] if len(g)]
        run = groups[:1] if sample_groups else groups
        t_layer = 0.0
        for gi, cells in enumerate(run):
            us = [lay["unit"][r] for r in cells]; ts = [lay["shared"][r] for r in cells]; fs = [lay["filter"][r] for r in cells]
            steps = sum(K for _, K in props)
            states = np.array([[O.pm_rng_state(1000 * li + gi * 10 + s, r) for s in range(steps)] for r in cells], dtype=np.uint64)
            lists = np.stack([[lab[u_[1], u_[0]]] * n_list for u_ in us]).astype(np.float32)
            t0 = time.perf_counter()
            ref.pm_group(us, ts, fs, props, 1, states, cost, lab, list_planes=lists)
            t_layer += time.perf_counter() - t0
            ran += 1
        total += t_layer * (len(groups) / len(run))
    ref.close()
    return total * 1e3, ran


def main():
    import torch
    import localexpstereo_b200 as L
    from localexpstereo_b200 import synth
    quick = "--quick" in sys.argv
    gpu, power = card()
    cores = os.cpu_count()
    for (W, H, D, windR) in [(450, 375, 64, 20), (2048, 1536, 256, 20)]:
        imL, imR = synth.synthetic_image(H, W, 42), synth.synthetic_image(H, W, 43)
        E = L.NaiveStereoEnergy(imL, imR, L.Parameters(lambda_=20, windR=windR, filterName="GF", filter_param1=1e-4), D - 1)
        ms_e, ms_g, evals, launches = device_pm(E, D, quick)
        ms_u, evals_u = device_unary(E, D, quick)
        base = dict(W=W, H=H, D=D, windR=windR, units=UNITS, gpu=gpu, power_limit=power)
        print(json.dumps(dict(what="naive_pm_iteration", proposers="V3_PROPOSERS_REFERENCE", launches=launches, ms_eager=round(ms_e, 3),
                              ms_graph=round(ms_g, 3), evals=evals, evals_per_s_graph=round(evals / (ms_g * 1e-3)), **base)), flush=True)
        print(json.dumps(dict(what="naive_unary_sweep", note="bench.py's naive workload: host-supplied planes, no proposals, no update",
                              ms=round(ms_u, 3), evals=evals_u, evals_per_s=round(evals_u / (ms_u * 1e-3)), **base)), flush=True)
        E.close()
        torch.cuda.empty_cache()
        from oracle import build_ref
        if build_ref.available() and not quick:
            sample = W * H > 1e6
            ms_r, ran = reference_pm(imL, imR, W, H, D, windR, sample)
            print(json.dumps(dict(what="reference_pm_iteration", host_cores=cores, groups_run=ran, extrapolated=sample, ms=round(ms_r, 1),
                                  note="oracle/_ref ref_pm_group per group, RANSAC slot replayed as a list", W=W, H=H, D=D, windR=windR)),
                  flush=True)


if __name__ == "__main__":
    main()
