"""Throughput of the bilateral filter ("BL") and the unfiltered mode ("") of the cost-volume energy on bench.py's workload
(2048 x 1536 x 256, windR 20, layers of unit 20 / 61 / 184 with 9 / 3 / 3 steps): one unary sweep (every group's steps through
Plan.eval_device into an H x W image in HBM) and one PatchMatch iteration (lexp_pm_sweep_iteration), timed with CUDA events.
Prints one JSON line per filter with evals/s, the card's name and its power limit (nvidia-smi, read only).  Not a test."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        return out
    except Exception as e:   # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--W", type=int, default=2048)
    ap.add_argument("--H", type=int, default=1536)
    ap.add_argument("--D", type=int, default=256)
    ap.add_argument("--windR", type=int, default=20)
    ap.add_argument("--filters", default="BL,")
    a = ap.parse_args()
    import torch
    import bench
    import localexpstereo_b200 as L
    from localexpstereo_b200.sweep import NativePMSweep
    W, H, D, windR = a.W, a.H, a.D, a.windR
    imL, vol = bench.make_inputs(W, H, D)
    units, steps = [20, 61, 184], [9, 3, 3]
    name_card = card()
    for name in a.filters.split(","):
        E = L.CostVolumeEnergy(imL, None, vol, None, L.Parameters(windR=windR, filterName=name, filter_param1=10.0, th_col=0.5), D - 1)
        lm = L.LayerManager(W, H, windR)
        plans, planes, evals = [], [], 0
        rng = np.random.default_rng(1)
        for li, u in enumerate(units):
            ly = lm.addLayer(u)
            for g in ly.disjointRegionSets:
                P = E.make_plan([ly.filterRegions[i] for i in g], [ly.sharedRegions[i] for i in g])
                pl = np.zeros((len(g), 4), np.float32)
                pl[:, 2] = rng.uniform(0, D - 1, len(g))
                plans.append((P, steps[li], torch.from_numpy(pl).cuda()))
                evals += P.filter_px * steps[li]
        out = torch.zeros((H, W), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        E.set_stream(s.cuda_stream)

        def sweep():
            for P, k, pl in plans:
                for _ in range(k):
                    P.eval_device(pl.data_ptr(), out.data_ptr(), W * 4, planes_on_device=True)
        sweep()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(s)
        sweep()
        t1.record(s)
        torch.cuda.synchronize()
        ms_unary = t0.elapsed_time(t1)
        S = NativePMSweep(E, unit_sizes=units, proposers=[[(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 8)], [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)],
                                                           [(L.PROP_EXPANSION, 1), (L.PROP_RANDOM, 2)]])
        S.begin()
        S.random_start(5)
        S.iteration(0, 1)
        torch.cuda.synchronize()
        t0.record(s)
        S.iteration(1, 2)
        t1.record(s)
        E.sync()
        torch.cuda.synchronize()
        ms_pm = t0.elapsed_time(t1)
        S.close()
        print(json.dumps({"filter": name, "workload": f"{W}x{H}x{D} windR {windR}", "evals_per_sweep": evals,
                          "unary_sweep_ms": ms_unary, "unary_evals_per_s": evals / (ms_unary * 1e-3),
                          "pm_iteration_ms": ms_pm, "card": name_card}), flush=True)
        for P, _, _ in plans:
            P.close()
        E.close()


if __name__ == "__main__":
    main()
